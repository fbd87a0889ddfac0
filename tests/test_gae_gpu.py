"""GPU: λ-returns (algorithm.gae_lambda, lambda_returns_kernel in csrc/a2c.cu) of IA2C, IPPO, MAA2C and MAPPO.

- The returns against the float64 mixture of n-step returns (tests/gae_ref.py) at λ in {0, 0.3, 0.95, 1}, γ in {0.9, 0.99}, T in {1, 31, 32,
  33, 64, 65, 500}, one and four agents, with and without standardise_returns, within 1e-5 of the batch's largest |R|.  These T are not the
  kernel's boundaries (lanes of 8 steps, windows of 256): tests/test_returns_edges_gpu.py sweeps those, row by row.
- Determinism, λ = 0 against the n_steps = 1 path, and the n-step path launching only nstep_returns_kernel while λ is unset.
- Full updates against the oracle with the λ-returns (MLP and GRU parts, shared, independent and SePS networks, the centralised critic, PPO chains
  of 4 epochs), and the reference's own A2CNetwork / PPONetwork at n_steps = 1 and T as λ = 0 and λ = 1.
- The drivers end to end (MAPPO on LBF, IPPO on RWARE at T = 500, eval from the saved config), and data-parallel training."""
import copy
import ctypes as C
import os
import types

import numpy as np
import pytest
import torch

from oracle import learner_ref as lr
from tests import gae_ref as gr
from tests import gru_ac_ref as gar
from tests.helpers import STRIDE, NearTie, TIE, ac_model, ac_oracle_batch, redraw_on_near_tie, reference_outputs, space, traj_store
from tests.test_rnn_ac_gpu import Case, Tracker, _batch, _check_update, _hp, _model, _oracle, _perturb_target

pytestmark = pytest.mark.gpu


def _ac(N, D, A, P, T, gamma=0.99, standardise=False, n_steps=5, lam=None, ppo=False, sharing=False):
    from codebase_b200.ac import model as M

    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=gamma, grad_clip=False, n_steps=n_steps, entropy_coef=0.001, value_loss_coef=0.5,
                                target_update_interval_or_tau=200, standardise_returns=standardise, num_epochs=4, ppo_clip=0.2, gae_lambda=lam)
    net = types.SimpleNamespace(layers=[128, 128], parameter_sharing=sharing, use_rnn=False, use_orthogonal_init=True, centralised=False)
    return (M.PPONetwork if ppo else M.A2CNetwork)([space(shape=(D,))] * N, [space(n=A)] * N, cfg, net, copy.copy(net), "cuda", max_envs=P,
                                                   max_episode_length=T)


def _episodes(rng, P, N, T, D, A=3):
    """P episodes of dense rewards: most end (done) before T, some run to T unterminated (truncated by the store)"""
    obs = (rng.integers(-1, 8, size=(P, N, T + 1, D)) / 4.0).astype(np.float32)
    act = rng.integers(0, A, size=(P, N, T)).astype(np.int32)
    rew = rng.standard_normal((P, N, T)).astype(np.float32)
    done = np.zeros((P, T + 1), np.uint8); filled = np.zeros((P, T), np.uint8)
    for e in range(P):
        end = int(rng.integers(1, T + 1)) if e % 3 else T
        filled[e, :end] = 1
        done[e, end] = 1 if end < T or e % 2 else 0
    return dict(obs=obs, act=act, rew=rew, done=done, filled=filled)


def _oracle_returns(s, vt, lam, gamma, ms=None):
    """float64 λ-returns (T, P, N) of a device-layout batch from the device's target values vt [N][P][T+1] (de-standardised with ms = (mean, var))"""
    v = vt.double().permute(2, 1, 0).numpy()
    if ms is not None:
        v = v * np.sqrt(ms[1].double().numpy()) + ms[0].double().numpy()
    rew = s["rew"].astype(np.float64).transpose(2, 0, 1)
    done = np.repeat(s["done"].astype(np.float64).T[:, :, None], rew.shape[2], axis=2)
    return gr.lambda_returns(rew, done, v, lam, gamma)


# ---- 1. the returns ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [1, 31, 32, 33, 64, 65, 500])
@pytest.mark.parametrize("N", [1, 4])
@pytest.mark.parametrize("standardise", [False, True], ids=["raw", "standardise"])
@pytest.mark.parametrize("gamma", [0.9, 0.99])
def test_returns_match_float64_oracle(T, N, standardise, gamma):
    P, D = 7, 5
    torch.manual_seed(T + N)
    m = _ac(N, D, 3, P, T, gamma=gamma, standardise=standardise, lam=0.5)
    m.theta_tgt.copy_(m.theta_tgt + 0.05 * torch.randn_like(m.theta_tgt))
    s = _episodes(np.random.default_rng(T * 10 + N), P, N, T, D)
    ts = traj_store(s, m.device)
    rms = lr.RunningMeanStdRef((N,)) if standardise else None
    if rms is not None:
        rms.mean, rms.var = rms.mean.double(), rms.var.double()
    for lam in (0.0, 0.3, 0.95, 1.0):
        m.set_gae_lambda(lam)
        ms = m.ret_ms()[:2] if standardise else None
        m.update_grads(ts, P)
        vt, ret, _ = m.scratch(P, T)
        want = _oracle_returns(s, vt.cpu(), float(np.float32(lam)), float(np.float32(gamma)), ms)
        if rms is not None:   # the running statistics absorb the returns, which are then standardised (ac/model.py:202-204)
            rms.update(torch.tensor(want))
            want = ((torch.tensor(want) - rms.mean) / torch.sqrt(rms.var)).numpy()
            mean, var, count = m.ret_ms()
            np.testing.assert_allclose(mean.numpy(), rms.mean.numpy(), rtol=1e-5, atol=1e-5)
            np.testing.assert_allclose(var.numpy(), rms.var.numpy(), rtol=1e-5, atol=1e-5)
        got = ret.double().permute(2, 1, 0).cpu().numpy()
        scale = float(np.abs(want).max())
        err = float(np.abs(got - want).max())
        assert err <= 1e-5 * scale, f"λ = {lam}: max error {err:.3e} vs largest |R| {scale:.3e}"
    m.close()


def test_set_gae_lambda_refuses_values_outside_0_1():
    from codebase_b200 import _native as nat

    m = _ac(2, 5, 3, 4, 10)
    for bad in (-0.001, 1.001, float("nan"), float("inf")):
        with pytest.raises(nat.NativeError, match="outside"):
            nat.check(m._lib.marl_a2c_set_gae_lambda(m._h, C.c_int32(1), C.c_float(bad)), "marl_a2c_set_gae_lambda")
        with pytest.raises(ValueError, match="gae_lambda"):
            m.set_gae_lambda(bad)
    nat.check(m._lib.marl_a2c_set_gae_lambda(m._h, C.c_int32(0), C.c_float(7.0)), "marl_a2c_set_gae_lambda")   # disabling ignores λ
    m.close()


def test_returns_are_deterministic():
    """two runs of the same update give the same bits: the returns, and the whole PPO state after two updates"""
    N, D, P, T = 4, 5, 16, 500
    torch.manual_seed(3)
    a = _ac(N, D, 3, P, T, lam=0.95, ppo=True)
    b = _ac(N, D, 3, P, T, lam=0.95, ppo=True)
    b.theta.copy_(a.theta); b.theta_tgt.copy_(a.theta_tgt)
    rng = np.random.default_rng(5)
    for step in (0, 1):
        ts = traj_store(_episodes(rng, P, N, T, D), a.device)
        rets = []
        for m in (a, b):
            m.update_from_store(ts, P, step)
            rets.append(m.scratch(P, T)[1].cpu().clone())
        assert torch.equal(rets[0], rets[1])
    for name in ("theta", "theta_tgt", "adam_m", "adam_v"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name
    a.close(); b.close()


@pytest.mark.parametrize("T", [1, 25, 500])
def test_lambda_zero_is_the_one_step_return(T):
    """λ = 0 (with n_steps = 5, unread) against the n-step path at n_steps = 1: the same returns to float32 rounding"""
    N, D, P = 2, 5, 32
    torch.manual_seed(T)
    a = _ac(N, D, 3, P, T, n_steps=1)
    b = _ac(N, D, 3, P, T, n_steps=5, lam=0.0)
    b.theta.copy_(a.theta); b.theta_tgt.copy_(a.theta_tgt)
    ts = traj_store(_episodes(np.random.default_rng(T), P, N, T, D), a.device)
    got = []
    for m in (a, b):
        m.update_grads(ts, P)
        got.append(m.scratch(P, T)[1].double().cpu())
    scale = float(got[0].abs().max())
    assert float((got[0] - got[1]).abs().max()) <= 2 * np.finfo(np.float32).eps * scale
    a.close(); b.close()


# Runs in a process of its own: a torch.profiler session is process state (CUPTI), and one left behind in the pytest process made a later
# test's profiler see no kernels at all.
LAUNCHES = r"""
import json, sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
from torch.profiler import ProfilerActivity, profile
from tests.helpers import traj_store
from tests.test_gae_gpu import _ac, _episodes

N, D, P, T = 2, 5, 32, 25
m = _ac(N, D, 3, P, T)
ts = traj_store(_episodes(np.random.default_rng(0), P, N, T, D), m.device)
m.update_grads(ts, P)   # warm-up
out = {}
for name, lam in (("unset", None), ("set", 0.95), ("unset_again", None)):
    m.set_gae_lambda(lam)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        m.update_grads(ts, P)
        torch.cuda.synchronize()
    out[name] = sorted({e.name for e in prof.events()})
m.close()
print(json.dumps(out))
"""


def test_nstep_path_launches_no_lambda_kernel():
    """gae_lambda unset: the update runs nstep_returns_kernel and never lambda_returns_kernel; set: the other way round; unset again: back"""
    import json
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, "-c", LAUNCHES, root], cwd=root, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-4000:]
    names = json.loads(p.stdout.strip().splitlines()[-1])
    for phase, runs, never in (("unset", "nstep_returns_kernel", "lambda_returns_kernel"), ("set", "lambda_returns_kernel", "nstep_returns_kernel"),
                               ("unset_again", "nstep_returns_kernel", "lambda_returns_kernel")):
        assert any(runs in n for n in names[phase]), (phase, names[phase])
        assert not any(never in n for n in names[phase]), (phase, names[phase])


# ---- 2. full updates against the oracle -----------------------------------------------------------------------------------------------------------
UPDATES = {
    "ia2c_mlp_indep": (Case(arnn=False, crnn=False, T=25, P=32), 0.95),
    "ia2c_mlp_shared_standardise": (Case(arnn=False, crnn=False, T=25, P=32, sharing=True, standardise=True, steps=(0, 3)), 0.3),
    "maa2c_mlp_central": (Case(arnn=False, crnn=False, T=25, P=32, centralised=True), 0.95),
    "ia2c_gru_seps": (Case(N=3, D=7, sharing=(0, 1, 0), T=7, P=24), 0.95),
    "maa2c_gru_central": (Case(T=7, P=32, centralised=True), 1.0),
    "ippo_mlp_chain": (Case(ppo=True, arnn=False, crnn=False, T=25, P=24, steps=(0, 3, 4), tu=2), 0.95),
    "mappo_mlp_chain_standardise": (Case(ppo=True, arnn=False, crnn=False, T=25, P=24, centralised=True, standardise=True, steps=(0, 3, 4), tu=2), 0.95),
    "ippo_gru_shared_chain": (Case(ppo=True, T=10, P=16, sharing=True, steps=(0, 3, 4), tu=2), 0.95),
}


@pytest.mark.parametrize("case", list(UPDATES))
@redraw_on_near_tie
def test_updates_match_oracle(case):
    c, lam = UPDATES[case]
    hp = _hp(c)
    m = _model(c)
    m.set_gae_lambda(lam)
    _perturb_target(m)
    st = _oracle(m, c)
    tr = Tracker(m.n_actor + m.n_critic)
    rng = np.random.default_rng(int(torch.randint(0, 1 << 30, (1,))))
    with gr.lambda_returns_in(float(np.float32(lam))):
        for u, step in enumerate(c.steps):
            s = _batch(c, rng)
            batch = ac_oracle_batch({k: v[: c.P] for k, v in s.items()})
            st0 = copy.deepcopy(st)
            want = gar.ppo_update(st, batch, hp, step, c.epochs, 0.2) if c.ppo else gar.a2c_update(st, batch, hp, step)
            if c.ppo and min(want["clip_margin"]) < TIE:
                raise NearTie(f"a ratio {min(want['clip_margin']):.1e} from the edge of the clip range")
            tgt0 = m.theta_tgt.cpu().numpy().copy()
            met = m.update_from_store(traj_store(s, m.device), c.P, step).cpu().numpy()
            _check_update(m, c, hp, st, st0, batch, want, met, step, tgt0, tr, f"{case} update {u}:")
    m.close()


@pytest.mark.parametrize("key", list(gr.GOLDEN_CASES))
def test_lambda_ends_match_the_reference_on_the_device(key):
    """the device at λ = 0 (resp. 1) against the reference's A2CNetwork / PPONetwork at n_steps = 1 (resp. T): returns, losses, statistics, parameters"""
    g = reference_outputs("gae_reference")
    cls, _, _, P, steps, epochs, clip, sharing, centralised, std, _, lam = gr.GOLDEN_CASES[key]
    hp = lr.A2CHP(grad_clip=float(clip or 0.0), target_update_interval_or_tau=2, n_steps=5)
    m = ac_model(hp, gr.N, gr.D, P, gr.T, A=gr.A, sharing=sharing, cls=cls, centralised=centralised, standardise=std, num_epochs=epochs)
    m.set_gae_lambda(lam)
    st = gr.golden_state(key)
    m.theta[: m.n_actor].copy_(st.actor); m.theta[m.n_actor:].copy_(st.critic); m.theta_tgt.copy_(st.target)
    tol = 2e-5 if cls == "PPONetwork" else 1e-5
    for u, (step, s) in enumerate(zip(steps, gr.golden_batches(key))):
        met = m.metrics_dict(m.update_from_store(traj_store(s, m.device), P, step))
        np.testing.assert_allclose([met[k] for k in gr.GOLDEN_METRICS], g[f"{key}_metrics"][u], rtol=tol, atol=tol)
        if u == 0 and not std:
            np.testing.assert_allclose(m.scratch(P, gr.T)[1].permute(2, 1, 0).cpu().numpy(), g[f"{key}_returns0"], rtol=1e-5, atol=1e-5)
    if std:
        mean, var, _ = m.ret_ms()
        np.testing.assert_allclose(mean.numpy(), g[f"{key}_ret_mean"], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(var.numpy(), g[f"{key}_ret_var"], rtol=1e-5, atol=1e-5)
    th, tg = m.theta.cpu().numpy(), m.theta_tgt.cpu().numpy()
    for got, name in ((th[: m.n_actor], "actor"), (th[m.n_actor:], "critic"), (tg, "target")):
        d = np.abs(got[::STRIDE] - g[f"{key}_{name}"])
        assert np.quantile(d, 0.999) < 1e-5 * max(1.0, tol / 1e-5), (name, d.max())
    m.close()


# ---- 3. the drivers -------------------------------------------------------------------------------------------------------------------------------
def test_mappo_driver_with_gae_and_eval(tmp_path, monkeypatch):
    import pandas as pd

    from codebase_b200 import eval as ev
    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    out = f"{tmp_path}/out"
    run.main(["+algorithm=mappo", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "algorithm.gae_lambda=0.95", "env.parallel_envs=256",
              "seed=1", "algorithm.total_steps=30000", "algorithm.eval_interval=6000", "algorithm.save_interval=6000", f"run_dir={out}"])
    df = pd.read_csv(f"{out}/results.csv")
    assert len(df) >= 3 and np.isfinite(df["loss"]).all() and np.isfinite(df["mean_episode_returns"]).all()
    monkeypatch.chdir(tmp_path)
    res = ev.main([f"path={out}", "episodes=16", "seed=3"])
    assert res["episodes"] == 16 and np.isfinite(res["mean_episode_returns"])


def test_ippo_rware_driver_with_gae_at_T500(tmp_path, monkeypatch):
    import pandas as pd

    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    run.main(["+algorithm=ippo", "env.name=rware:rware-tiny-4ag-v2", "env.time_limit=500", "algorithm.gae_lambda=0.95", "env.parallel_envs=32", "seed=2",
              "algorithm.total_steps=64000", "algorithm.eval_interval=16000", f"run_dir={tmp_path}/out"])
    df = pd.read_csv(tmp_path / "out" / "results.csv")
    assert len(df) >= 2 and np.isfinite(df["loss"]).all() and np.isfinite(df["value_loss"]).all()


def test_two_handles_with_summed_grads_match_the_union_batch():
    """data-parallel PPO with λ-returns, two ranks emulated on one device: the ranks stay bit-identical and match one handle on the union batch"""
    from tests import test_distributed_gpu as td

    envs = [td._env(0), td._env(td.P)]
    torch.manual_seed(0)

    def make(max_envs):
        m = td._ac(True, envs[0], max_envs)
        m.set_gae_lambda(0.95)
        return m

    ranks = [make(td.P) for _ in range(2)]
    union = make(2 * td.P)
    for m in (ranks[1], union):
        td._copy_params(m, ranks[0])
    for step in (0, 3200):
        halves, ub = td._ac_batches(ranks[0], envs)
        for e in range(ranks[0].num_epochs):
            for r in range(2):
                ranks[r].epoch_grads(halves[r], td.P, e)
            td._sum_into([(ranks[0].grad, ranks[1].grad)])
            met = [m.epoch_apply(step, e).clone() for m in ranks]
        want = union.update_from_store(ub, 2 * td.P, step)
        assert torch.equal(met[0], met[1])
        for k in (0, 2, 3):
            assert abs(float(met[0][k]) - float(want[k])) <= 1e-4 * max(1.0, abs(float(want[k]))), k
    for name in ("theta", "theta_tgt", "adam_m", "adam_v"):
        assert torch.equal(getattr(ranks[0], name), getattr(ranks[1], name)), name
    td._close(ranks[0].theta, union.theta, "theta")


def test_torchrun_two_ranks_on_one_device(tmp_path):
    """`torchrun -m codebase_b200.run ... algorithm.gae_lambda=0.95` with two ranks on one device: the ranks end with the same parameters and count the
    same global env steps; one rank under torchrun reproduces the plain single-process run bit for bit"""
    import pandas as pd

    from tests import test_distributed_gpu as td

    job = lambda out: ["+algorithm=mappo", f"env.name={td.LBF}", "env.time_limit=25", "env.parallel_envs=32", "algorithm.gae_lambda=0.95", "seed=3",   # noqa: E731
                       "algorithm.total_steps=8000", "algorithm.eval_interval=1600", "algorithm.save_interval=1600", f"run_dir={out}"]
    two = tmp_path / "two"; two.mkdir()
    (h0, local0, global0), (h1, local1, global1) = [h.read_text().split() for h in td._launch(two, 2, job(two / "out"))]
    assert h0 == h1 and global0 == global1 and int(global0) == int(local0) + int(local1)
    assert np.isfinite(pd.read_csv(two / "out" / "results.csv")["loss"]).all()
    a, b = tmp_path / "a", tmp_path / "b"
    a.mkdir(); b.mkdir()
    ha = td._launch(a, 1, job(a / "out"), torchrun=False)
    hb = td._launch(b, 1, job(b / "out"), torchrun=True)
    assert ha[0].read_text() == hb[0].read_text()
    da, db = pd.read_csv(a / "out" / "results.csv"), pd.read_csv(b / "out" / "results.csv")
    cols = [c for c in da.columns if "episode_time" not in c]
    pd.testing.assert_frame_equal(da[cols], db[cols])
    assert os.path.exists(two / "out" / "config.yaml")

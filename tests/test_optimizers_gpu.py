"""GPU: algorithm.optimizer = AdamW / RMSprop / Adagrad / SGD in every learner, against the oracle (tests/optim_ref.py: torch.optim's steps,
pinned bitwise to torch.optim by tests/test_optimizers.py) over chains of updates that are never re-synchronised with it.

- IDQN on both training paths (tensor-core pipeline, fused FP32 kernel), through the fused tail and the two-kernel tail; VDN with a shared
  network; QMIX (agents' networks and mixer, one optimiser, the mixer unclipped); recurrent IDQN.
- IA2C, MAPPO (centralised critic, 4 epochs, clipped), recurrent IA2C.
- update_n bit for bit against the update_from_store loop it replaces, on two handles; the tensor-core images kept current by the step (equal to a
  full repack, and the tensor-core forward equal to the FP32 forward); two A2C handles ending bit-identical; set_optimizer refused after a step.
- One short training run per family from the command line, and the two-GPU peer exchange with RMSprop (skipped on a one-GPU box)."""
import copy
import ctypes as C
import dataclasses
import os
import types

import numpy as np
import pytest
import torch

from oracle import gru_ref as gr
from oracle import learner_ref as lr
from oracle import policy_ref
from oracle import qmix_ref as qr
from tests import gru_ac_ref as gar
from tests import optim_ref as orf
from tests.helpers import ac_batch, ac_oracle_batch, assert_grad_close, close_scaled, random_store, space, traj_store

pytestmark = pytest.mark.gpu
A = 6
OPTS = ("AdamW", "RMSprop", "Adagrad", "SGD")
MIXING = dict(embed_dim=64, hypernet_layers=2, hypernet_embed=32)   # the QMIX oracle's mixer
SEED = 0x0971_3A11
# largest |step| / lr of one optimiser step per element (Adam and AdamW: ~1; RMSprop: g / sqrt((1 - alpha) g^2) = 10 on the first step; Adagrad: 1;
# SGD: |g| <= 1 after clipping at 1): the bound of an element whose gradient is too small to judge, as in tests/test_update_chain_gpu.py
STEP = {"AdamW": 1.0, "RMSprop": 10.0, "Adagrad": 1.0, "SGD": 1.0}


def _opt(name, on):
    from codebase_b200 import _native as nat

    nat.check(nat.lib().marl_set_option(name, C.c_int32(int(on))), "marl_set_option")


@pytest.fixture(autouse=True)
def _restore():
    yield
    _opt(b"tensor_core_backward", True)   # the library defaults
    _opt(b"tensor_core_forward", True)


@dataclasses.dataclass(frozen=True)
class DqnCase:
    mixer: int = 0
    N: int = 2
    D: int = 15
    sharing: bool = False
    B: int = 48
    T: int = 12
    K: int = 3
    rnn: bool = False
    tc_backward: bool = True
    cap: int = 200
    double_q: bool = False   # (double-Q near-ties are covered elsewhere; the reference fixture's cases use it)
    obs_scale: float = 1.0   # QMIX: observations / 10 -- at full scale the unclipped mixer's first SGD step diverges (loss 2e5, then NaN),
                             # as it does in the reference


DQN_CASES = {
    "idqn2_fused_tail": DqnCase(),                              # tensor-core training pass, fused reduce + step tail
    "idqn2_fp32_train": DqnCase(tc_backward=False),             # the fused FP32 training kernel
    "idqn4_two_kernel_tail": DqnCase(N=4),                      # grad_reduce_kernel + adam_kernel<OPT>
    "vdn3_shared": DqnCase(mixer=1, N=3, sharing=True),
    "qmix2": DqnCase(mixer=2, B=32, T=10, obs_scale=0.1),                      # the mixer's step: adam_kernel<OPT>, unclipped
    "idqn2_rnn": DqnCase(rnn=True, B=16, T=10),
}


def _dqn_hp(c):
    # grad_clip 1.0; hard target sync every 2 updates (the chain crosses one)
    return lr.DqnHP(grad_clip=1.0, double_q=c.double_q, target_update_interval_or_tau=2, mixer=c.mixer)


def _dqn(c, opt):
    from codebase_b200.dqn import model as M

    hp = _dqn_hp(c)
    cfg = types.SimpleNamespace(optimizer=opt, lr=hp.lr, gamma=hp.gamma, grad_clip=hp.grad_clip, double_q=hp.double_q,
                                target_update_interval_or_tau=hp.target_update_interval_or_tau, standardise_returns=False)
    args = ([space(shape=(c.D,))] * c.N, [space(n=A)] * c.N, cfg, [128, 128], c.sharing, c.rnn, True)
    if c.mixer == 2:
        return M.QMixNetwork(*args, MIXING, "cuda", max_batch=c.B, max_episode_length=c.T)
    return (M.VDNetwork if c.mixer else M.QNetwork)(*args, "cuda", max_batch=c.B, max_episode_length=c.T)


def _perturb_target(m):
    m.theta_tgt.copy_(m.theta + 0.01 * torch.randn_like(m.theta))
    if m.mixer == 2:
        m.mix_tgt.copy_(m.mix + 0.01 * torch.randn_like(m.mix))
    m.params_changed()


def _state_close(opt, got, want_m, want_v, tol, what):
    """the optimiser state of the device (optimizer_state(): torch's names) against the oracle's m / v buffers"""
    names = dict(zip(orf.STATE[opt], (want_m, want_v)))
    assert set(got) == {k for k in names if k is not None}, (what, sorted(got))
    for k, t in got.items():
        close_scaled(t.cpu().numpy(), names[k].numpy(), tol if k == "exp_avg" else 2 * tol)


def _params_close(mine, theirs, u, hp, opt, tol, what):
    d = np.abs(mine.cpu().numpy() - theirs.numpy())
    assert np.quantile(d, 0.999) < tol and d.max() < 2 * STEP[opt] * hp.lr * (u + 1) + 1e-6, (what, np.quantile(d, 0.999), d.max())


@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("case", list(DQN_CASES))
def test_dqn_chain_matches_oracle(case, opt):
    """K updates through marl_dqn_update (update_from_store); after each: gradient, loss, optimiser state, parameters and targets against the
    oracle, which steps in place beside the device and is never copied back"""
    c = DQN_CASES[case]
    _opt(b"tensor_core_backward", c.tc_backward)
    torch.manual_seed(17)
    hp = _dqn_hp(c)
    m = _dqn(c, opt)
    assert m.optimizer_name == opt
    _perturb_target(m)
    nets = list(m.agent_net)
    if c.mixer == 2:
        st = qr.QmixState(m.theta.cpu().clone(), m.theta_tgt.cpu().clone(), m.mix.cpu().clone(), m.mix_tgt.cpu().clone(), nets, c.D, A)
    else:
        st = lr.DqnState(m.theta.cpu().clone(), m.theta_tgt.cpu().clone(), nets, c.D, A)
    s = random_store(np.random.default_rng(c.B + 7 * c.N), c.cap, c.N, c.T, c.D, c.mixer != 0)
    s["obs"] *= c.obs_scale
    ts = traj_store(s, m.device)
    n = m.n_params
    gtol = 2e-5 if c.mixer == 2 else 1e-5
    stol = 5e-5 if c.rnn else gtol   # optimiser state: the GRU kernels' bars of tests/test_rnn_dqn_gpu.py
    for u in range(c.K):
        what = f"{opt} update {u}:"
        idx = policy_ref.replay_sample(SEED, u, c.B, c.cap)
        batch = lr.batch_from_store(s, idx)
        st0 = copy.deepcopy(st)
        with orf.optimizer(opt):
            if c.mixer == 2:
                want, risk = qr.qmix_update(st, batch, hp), (lambda: qr.qmix_kink_risk(st0, batch, hp))
            elif c.rnn:
                want, risk = gr.dqn_update(st, batch, hp), (lambda: gr.dqn_kink_risk(st0, batch, hp))
            else:
                want, risk = lr.dqn_update(st, batch, hp), None
        met = m.update_from_store(ts, torch.tensor(idx, device=m.device)).cpu().numpy()
        g = m.grad.cpu().numpy()
        assert_grad_close(lr, st0, batch, hp, g[:n] / g[n + 1], want["grad"].numpy(), tol=gtol, what=what, kink_risk=risk)
        assert abs(met[0] - want["loss"]) <= 1e-5 * max(1.0, abs(want["loss"])), (what, met[0], want["loss"])
        state = m.optimizer_state()
        _state_close(opt, {k: t for k, t in state.items() if not k.startswith("mixer.")}, st.m, st.v, stol, what)
        pairs = [("theta", m.theta, st.theta), ("theta_tgt", m.theta_tgt, st.theta_tgt)]
        if c.mixer == 2:
            _state_close(opt, {k[6:]: t for k, t in state.items() if k.startswith("mixer.")}, st.mix_m, st.mix_v, stol, what + " mixer")
            pairs += [("mix", m.mix, st.mix), ("mix_tgt", m.mix_tgt, st.mix_tgt)]
        for name, mine, theirs in pairs:
            _params_close(mine, theirs, u, hp, opt, 2e-5 if c.mixer == 2 else 1e-5, f"{what} {name}")
    m.close()


@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("case", ["idqn2_fused_tail", "qmix2"])
def test_update_n_is_the_loop_it_replaces(case, opt):
    """update_n (the fused tail, next indices drawn in it) on one handle, replay_sample + update_from_store on a second handle with the same
    parameters: every buffer ends equal bit for bit"""
    from codebase_b200 import _native as nat

    c = dataclasses.replace(DQN_CASES[case], K=5)
    torch.manual_seed(3)
    a = _dqn(c, opt)
    _perturb_target(a)
    b = _dqn(c, opt)
    b.theta.copy_(a.theta); b.theta_tgt.copy_(a.theta_tgt)
    if c.mixer == 2:
        b.mix.copy_(a.mix); b.mix_tgt.copy_(a.mix_tgt)
    b.params_changed()
    s = random_store(np.random.default_rng(5), c.cap, c.N, c.T, c.D, c.mixer != 0)
    s["obs"] *= c.obs_scale
    ts = traj_store(s, a.device)
    a.update_n(ts, c.B, c.cap, SEED, 0, c.K)
    idx = torch.zeros(c.B, dtype=torch.int32, device=b.device)
    for u in range(c.K):
        nat.check(nat.lib().marl_replay_sample(C.c_uint64(SEED), C.c_uint64(u), C.c_int32(c.B), C.c_int32(c.cap), nat.ptr(idx), nat.stream_ptr()), "sample")
        b.update_from_store(ts, idx)
    names = ["theta", "theta_tgt", "adam_m", "adam_v", "grad", "_metrics"] + (["mix", "mix_tgt", "mix_m", "mix_v"] if c.mixer == 2 else [])
    for k in names:
        x, y = getattr(a, k).cpu(), getattr(b, k).cpu()
        assert torch.equal(x, y), (opt, k, float((x - y).abs().max()))
    a.close(); b.close()


@pytest.mark.parametrize("opt", ["RMSprop", "AdamW"])
def test_step_keeps_tensor_core_images_current(opt):
    """after a chain of fused updates the images the step rewrote parameter by parameter are what a full repack makes (bitwise), and the
    tensor-core forward equals the FP32 forward"""
    c = DQN_CASES["idqn2_fused_tail"]
    torch.manual_seed(5)
    m = _dqn(c, opt)
    _perturb_target(m)
    ts = traj_store(random_store(np.random.default_rng(77), c.cap, c.N, c.T, c.D, False), m.device)
    m.update_n(ts, c.B, c.cap, SEED, 0, 5)
    obs = torch.tensor(np.random.default_rng(78).integers(-1, 12, size=(257, c.N, c.D)), dtype=torch.float32, device=m.device)
    idx = torch.tensor(policy_ref.replay_sample(SEED, 5, c.B, c.cap), device=m.device)

    def outputs():
        q = m.q_values(obs).clone()
        m.update_grads(ts, idx)
        return dict(q=q.cpu(), grad=m.grad.cpu().clone())

    kept = outputs()
    _opt(b"tensor_core_forward", False)
    fp32 = m.q_values(obs).cpu()
    _opt(b"tensor_core_forward", True)
    m.params_changed()
    repacked = outputs()
    for k in kept:
        assert torch.equal(kept[k], repacked[k]), (k, float((kept[k] - repacked[k]).abs().max()))
    assert torch.allclose(kept["q"], fp32, rtol=1e-5, atol=1e-5), float((kept["q"] - fp32).abs().max())
    m.close()


def test_set_optimizer_is_refused_after_a_step():
    from codebase_b200 import _native as nat
    from codebase_b200 import optimizers

    c = DQN_CASES["idqn2_fused_tail"]
    m = _dqn(c, "RMSprop")
    ts = traj_store(random_store(np.random.default_rng(1), c.cap, c.N, c.T, c.D, False), m.device)
    optimizers.apply(m._lib, "marl_dqn_set_optimizer", m._h, "SGD")   # still allowed: no step yet
    m.update_n(ts, c.B, c.cap, SEED, 0, 1)
    with pytest.raises(nat.NativeError, match="already taken an optimiser step"):
        optimizers.apply(m._lib, "marl_dqn_set_optimizer", m._h, "Adam")
    bad = nat.Optimizer(7, 0.9, 0.999, 0.0, 1e-8, 0.0)
    assert nat.lib().marl_dqn_set_optimizer(m._h, C.byref(bad)) == -1
    m.close()
    a = _ac(AC_CASES["ia2c2"], "Adagrad")
    optimizers.apply(a._lib, "marl_a2c_set_optimizer", a._h, "Adagrad")
    _ac_update(a, traj_store(ac_batch(np.random.default_rng(2), 16, 2, 10, 15), a.device), 16, 0)
    with pytest.raises(nat.NativeError, match="already taken an optimiser step"):
        optimizers.apply(a._lib, "marl_a2c_set_optimizer", a._h, "SGD")
    a.close()


# ---- actor-critic ----------------------------------------------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class AcCase:
    ppo: bool = False
    N: int = 2
    D: int = 15
    centralised: bool = False
    sharing: bool = False
    rnn: bool = False
    P: int = 16
    T: int = 10
    steps: tuple = (0, 2, 3)      # target sync at step % 2 == 0
    grad_clip: float = 0.0
    epochs: int = 4


AC_CASES = {
    "ia2c2": AcCase(),
    "mappo2_centralised_clip": AcCase(ppo=True, centralised=True, grad_clip=0.5),
    "ia2c2_rnn": AcCase(rnn=True),
}


def _ac_hp(c):
    return lr.A2CHP(grad_clip=c.grad_clip, target_update_interval_or_tau=2)


def _ac(c, opt):
    from codebase_b200.ac import model as M

    hp = _ac_hp(c)
    cfg = types.SimpleNamespace(optimizer=opt, lr=hp.lr, gamma=hp.gamma, grad_clip=hp.grad_clip, n_steps=hp.n_steps, entropy_coef=hp.entropy_coef,
                                value_loss_coef=hp.value_loss_coef, target_update_interval_or_tau=hp.target_update_interval_or_tau,
                                standardise_returns=False, num_epochs=c.epochs, ppo_clip=0.2)
    net = types.SimpleNamespace(layers=[128, 128], parameter_sharing=c.sharing, use_rnn=c.rnn, use_orthogonal_init=True, centralised=False)
    cnet = types.SimpleNamespace(**{**vars(net), "centralised": c.centralised})
    cls = M.PPONetwork if c.ppo else M.A2CNetwork
    return cls([space(shape=(c.D,))] * c.N, [space(n=A)] * c.N, cfg, net, cnet, "cuda", max_envs=c.P, max_episode_length=c.T)


def _ac_update(m, ts, n_envs, step):
    """one update; its metrics as a dict (loss, actor_loss, value_loss, entropy)"""
    return m.metrics_dict(m.update_from_store(ts, n_envs, step))


@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("case", list(AC_CASES))
def test_ac_chain_matches_oracle(case, opt):
    """K A2C / PPO updates on the device beside the oracle: metrics after every update; optimiser state, parameters and target critic"""
    c = AC_CASES[case]
    torch.manual_seed(23)
    hp = _ac_hp(c)
    m = _ac(c, opt)
    m.theta_tgt.copy_(m.theta_tgt + 0.01 * torch.randn_like(m.theta_tgt))
    st = lr.A2CState(m.theta[: m.n_actor].cpu().clone(), m.theta[m.n_actor:].cpu().clone(), m.theta_tgt.cpu().clone(), list(m.actor_net),
                     list(m.critic_net), c.D, A, centralised=c.centralised)
    rng = np.random.default_rng(31)
    tol = 2e-5 if c.ppo else 1e-5
    for u, step in enumerate(c.steps):
        what = f"{opt} update {u}:"
        s = ac_batch(rng, c.P, c.N, c.T, c.D)
        batch = ac_oracle_batch(s)
        with orf.optimizer(opt):
            if c.rnn:
                want = gar.ppo_update(st, batch, hp, step, c.epochs, 0.2) if c.ppo else gar.a2c_update(st, batch, hp, step)
            else:
                want = lr.ppo_update(st, batch, hp, step, c.epochs, 0.2) if c.ppo else lr.a2c_update(st, batch, hp, step)
        met = _ac_update(m, traj_store(s, m.device), c.P, step)
        assert abs(met["loss"] - want["loss"]) <= tol * max(1.0, abs(want["loss"])), (what, met["loss"], want["loss"])
        state = m.optimizer_state()
        want_m, want_v = torch.cat([st.m["actor"], st.m["critic"]]), torch.cat([st.v["actor"], st.v["critic"]])
        _state_close(opt, state, want_m, want_v, 2 * tol, what)   # (PPO: four steps per update)
        _params_close(m.theta, torch.cat([st.actor, st.critic]), u if not c.ppo else c.epochs * (u + 1) - 1, hp, opt, tol, f"{what} theta")
        _params_close(m.theta_tgt, st.target, u if not c.ppo else c.epochs * (u + 1) - 1, hp, opt, tol, f"{what} target")
    m.close()


@pytest.mark.parametrize("opt", ["RMSprop", "AdamW"])
def test_two_ac_handles_end_bit_identical(opt):
    c = AC_CASES["mappo2_centralised_clip"]
    torch.manual_seed(41)
    a = _ac(c, opt)
    b = _ac(c, opt)
    b.theta.copy_(a.theta); b.theta_tgt.copy_(a.theta_tgt)
    rng = np.random.default_rng(43)
    for step in c.steps:
        ts = traj_store(ac_batch(rng, c.P, c.N, c.T, c.D), a.device)
        _ac_update(a, ts, c.P, step); _ac_update(b, ts, c.P, step)
    for k in ("theta", "theta_tgt", "adam_m", "adam_v", "grad"):
        assert torch.equal(getattr(a, k).cpu(), getattr(b, k).cpu()), (opt, k)
    a.close(); b.close()


# ---- command line ----------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("alg,opt", [("qmix", "RMSprop"), ("mappo", "AdamW")])
def test_driver_trains_with_the_optimizer(tmp_path, monkeypatch, alg, opt):
    import pandas as pd

    from codebase_b200 import run

    monkeypatch.chdir(tmp_path)
    extra = ["algorithm.batch_size=128", "algorithm.buffer_size=4096", "algorithm.updates_per_iteration=16"] if alg == "qmix" else []
    run.main([f"+algorithm={alg}", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "env.parallel_envs=256", "seed=0",
              f"algorithm.optimizer={opt}", "algorithm.total_steps=60000", "algorithm.eval_interval=20000", f"run_dir={tmp_path}/out"] + extra)
    df = pd.read_csv(tmp_path / "out" / "results.csv")
    losses = [k for k in df.columns if k.endswith("loss")]
    assert len(df) >= 2 and losses, list(df.columns)
    for k in losses:
        assert np.isfinite(df[k].to_numpy()).all(), (k, df[k].to_numpy())


# ---- two GPUs --------------------------------------------------------------------------------------------------------------------------------------
def _peer_worker(rank, world, port, out):
    import torch.distributed as dist

    from codebase_b200.dqn import model as M
    from codebase_b200.lbf import TrajStore

    N, D, T, B = 2, 15, 25, 96
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    torch.cuda.set_device(rank)
    cfg = types.SimpleNamespace(optimizer="RMSprop", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=2,
                                standardise_returns=False)

    def make():
        m = M.QNetwork([space(shape=(D,))] * N, [space(n=A)] * N, cfg, [128, 128], False, False, True, f"cuda:{rank}", max_batch=B, max_episode_length=T)
        rng0 = np.random.default_rng(1234)
        m.theta.copy_(torch.as_tensor(0.05 * rng0.standard_normal(m.theta.numel()), dtype=torch.float32).view_as(m.theta))
        m.params_changed(); m.hard_update()
        return m

    rng = np.random.default_rng(100 + rank)
    ts = TrajStore(200, N, T, D, torch.device(f"cuda:{rank}"))
    ts.obs.copy_(torch.as_tensor(rng.integers(-1, 9, size=tuple(ts.obs.shape)).astype(np.float32)))
    ts.act.copy_(torch.as_tensor(rng.integers(0, A, size=tuple(ts.act.shape)).astype(np.int32)))
    ts.rew.copy_(torch.as_tensor((rng.random(tuple(ts.rew.shape)) < 0.3).astype(np.float32)))
    ts.filled.fill_(1)
    idx = [torch.tensor(rng.integers(0, 200, size=B).astype(np.int32), device=f"cuda:{rank}") for _ in range(3)]
    peer = make()
    peer.attach_peers()
    for k in range(3):
        peer.update_from_store(ts, idx[k])
    torch.cuda.synchronize()
    ref = make()
    for k in range(3):
        ref.update_grads(ts, idx[k])
        g = ref.grad.cpu()
        dist.all_reduce(g)
        ref.grad.copy_(g)
        ref.update_apply()
    torch.cuda.synchronize()
    th = peer.theta.cpu()
    gathered = [torch.empty_like(th) for _ in range(world)]
    dist.all_gather(gathered, th)
    out.put((rank, not peer.peer_timed_out(), bool(all(torch.equal(gathered[0], t) for t in gathered)), float((th - ref.theta.cpu()).abs().max()),
             float((peer.adam_v.cpu() - ref.adam_v.cpu()).abs().max() / max(float(ref.adam_v.abs().max()), 1e-30))))
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs on one node")
def test_peer_exchange_with_rmsprop():
    """RMSprop through the in-kernel exchange (reduce_adam_kernel<1, RMSprop>) against update_grads + all-reduce + update_apply"""
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    procs = [ctx.Process(target=_peer_worker, args=(r, 2, 29631, out)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=240)
    hung = [p for p in procs if p.is_alive()]
    for p in hung:
        p.kill()
    assert not hung, "a rank did not finish"
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    for rank, healthy, same, d_theta, d_v in [out.get(timeout=10) for _ in range(2)]:
        assert healthy and same, rank
        assert d_theta <= 1e-5 and d_v <= 1e-5, (rank, d_theta, d_v)


# ---- the reference's own classes (tests/golden/optimizers_reference.npz) through the C ABI -----------------------------------------------------------
def _device_record(m, grad_clip, fam):
    """(loss-free) flat device state after an update, in the fixture's order: the gradient the step consumed (after the clip), parameters, target,
    optimiser state by torch's names"""
    from tests.helpers import clipped

    g = m.grad.cpu().numpy()
    n = m.n_params if hasattr(m, "n_params") else m.n_actor + m.n_critic
    fill = g[n + 1]
    grad = clipped(g[:n] / fill, grad_clip)
    theta, target = m.theta.cpu().numpy(), m.theta_tgt.cpu().numpy()
    state = {k: t.cpu().numpy() for k, t in m.optimizer_state().items()}
    if fam == "QMixNetwork":   # the mixer after the agents' networks, unclipped
        grad = np.concatenate([grad, m.mix_grad[: m.n_mix].cpu().numpy() / fill])
        theta, target = np.concatenate([theta, m.mix.cpu().numpy()]), np.concatenate([target, m.mix_tgt.cpu().numpy()])
        state = {k: np.concatenate([t, state[f"mixer.{k}"]]) for k, t in state.items() if not k.startswith("mixer.")}
    return dict(grad=grad, theta=theta, target=target, **state)


# MAPPO with AdamW or RMSprop on the device: the first update only.  Their first step moves a parameter by lr (AdamW) or 10 lr (RMSprop) whatever
# its gradient's size, so where the device's gradient (2e-5 from the oracle's for PPO, tests/test_ppo.py) and the reference's straddle zero the
# move flips, and the next update's four epochs start from parameters that differ by lr there.  Measured on an H100: after update 1 AdamW's
# exp_avg is 1.1e-4 of its scale from the reference's (0.999 quantile); with RMSprop the loss of update 2 is 1.2e-4 (relative) from it.  The
# CPU oracle, which rounds as the reference does, matches all three updates (tests/test_optimizers.py).
DEVICE_UPDATES = {("mappo", "AdamW"): range(1), ("mappo", "RMSprop"): range(1)}


@pytest.mark.parametrize("opt", OPTS)
@pytest.mark.parametrize("key", ["idqn", "vdn_shared", "qmix", "idqn_rnn", "ia2c", "maa2c", "mappo", "ia2c_rnn"])
def test_reference_fixture_on_device(key, opt):
    """the fixture's cases (seeded weights, the same batches) on the device: loss, clipped gradient, parameters, optimiser state and target
    after every update against what the reference's QNetwork / VDNetwork / QMixNetwork / A2CNetwork / PPONetwork (MLP and GRU) computed with
    torch.optim.<opt>"""
    from tests import test_optimizers as cpu
    from tests.helpers import reference_outputs

    g = reference_outputs("optimizers_reference")
    stride = int(g[f"{key}_stride"])
    rc = cpu.REF_CASES[key]
    st, hp = cpu._ref_case(key)
    if cpu.is_dqn(rc):
        c = DqnCase(mixer=("QNetwork", "VDNetwork", "QMixNetwork").index(rc.fam), N=rc.N, D=rc.D, sharing=rc.sharing, B=cpu.REF_B, T=cpu.REF_T,
                    cap=64, double_q=hp.double_q, rnn=rc.rnn)
        m = _dqn(c, opt)
        m.theta.copy_(st.theta); m.theta_tgt.copy_(st.theta_tgt)
        if rc.fam == "QMixNetwork":
            m.mix.copy_(st.mix); m.mix_tgt.copy_(st.mix_tgt)
        m.params_changed()
    else:
        c = AcCase(ppo=rc.fam == "PPONetwork", N=rc.N, D=rc.D, centralised=rc.central, sharing=rc.sharing, rnn=rc.rnn, P=cpu.REF_B, T=cpu.REF_T,
                   grad_clip=rc.grad_clip, epochs=cpu.REF_EPOCHS)
        m = _ac(c, opt)
        m.theta.copy_(torch.cat([st.actor, st.critic])); m.theta_tgt.copy_(st.target)
    loose = rc.fam in ("PPONetwork", "QMixNetwork") or rc.rnn
    tol = 2e-5 if loose else 1e-5
    # optimiser state relative to its scale: twice the gradient's bar (v ~ g^2), and the GRU bar of tests/test_optimizers.py
    stol = 5e-5 if rc.rnn else 2 * tol
    for u, (_, s, idx) in enumerate(cpu._ref_batches(key)):
        if u not in DEVICE_UPDATES.get((key, opt), range(cpu.REF_UPDATES)):
            break
        p = f"{key}_{opt}_{u}"
        if idx is None:
            loss = _ac_update(m, traj_store(s, m.device), cpu.REF_B, u)["loss"]
        else:
            loss = float(m.update_from_store(traj_store(s, m.device), torch.tensor(idx, dtype=torch.int32, device=m.device))[0])
        want = float(g[f"{p}_loss"])
        assert abs(loss - want) <= tol * max(1.0, abs(want)), (p, loss, want)
        rec = _device_record(m, hp.grad_clip, rc.fam)
        want_g = g[f"{p}_grad"]
        dg = np.abs(rec["grad"][::stride] - want_g)
        assert np.quantile(dg, 0.999) <= tol * max(1.0, float(np.abs(want_g).max())), (p, "grad", dg.max())
        for name in ("theta", "target"):
            d = np.abs(rec[name][::stride] - g[f"{p}_{name}"])
            assert np.quantile(d, 0.999) < tol, (p, name, d.max())
        assert {k for k in rec if k not in ("grad", "theta", "target")} == {k for k in orf.STATE[opt] if k is not None}, (p, sorted(rec))
        for name in orf.STATE[opt]:
            if name is not None:
                want_s = g[f"{p}_{name}"]
                d = np.abs(rec[name][::stride] - want_s)
                assert np.quantile(d, 0.999) <= stol * max(float(np.abs(want_s).max()), 1e-30), (p, name, np.quantile(d, 0.999))
    m.close()

"""GPU, one device is enough: data-parallel training (codebase_b200/distributed.py and the drivers) and the per-epoch PPO split.

- In-process emulation of two ranks: two handles on one GPU with different data, the exchanged buffers summed with torch between update_grads and
  update_apply.  The two handles stay bit-identical and match one handle updated on the union batch.
- marl_ppo_update against marl_ppo_prepare + K x (marl_ppo_epoch_grads + marl_ppo_epoch_apply), bit for bit.
- Env shards with env_gid0 = 0 and P collect exactly the two halves of one env set of 2P.
- torchrun with two ranks on this one device (gloo, the all-reduce between the two calls): one results.csv, one set of checkpoints, the global
  env-step count, bit-identical parameters on both ranks; and torchrun with one rank reproduces a plain run.
- Two devices (skipped otherwise): one torchrun run per learner family."""
import os
import signal
import socket
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T, P = 25, 64
LBF = "lbforaging:Foraging-8x8-2p-3f-v3"


def _env(gid0, n=P, name=LBF, time_limit=T):
    from codebase_b200.utils.envs import make_env

    return make_env(7, name=name, time_limit=time_limit, parallel_envs=n, env_gid0=gid0)


def _copy_params(dst, src):
    for name in ("theta", "theta_tgt", "mix", "mix_tgt"):
        if getattr(src, name, None) is not None:
            getattr(dst, name).copy_(getattr(src, name))
    if hasattr(dst, "params_changed"):
        dst.params_changed()


def _sum_into(pairs):
    """The all-reduce of two ranks, done with torch: both buffers end with the sum."""
    for a, b in pairs:
        s = a + b
        a.copy_(s)
        b.copy_(s)


def _close(got, want, what):
    d = (got - want).abs()
    assert float(d.quantile(0.999)) < 1e-5 and float(d.max()) < 2e-3, f"{what}: max {float(d.max())}"


# ---- DQN family ------------------------------------------------------------------------------------------------------------------------------
def _dqn(kind, B, rnn, env):
    from codebase_b200.dqn import model as M

    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=2, standardise_returns=False)
    args = (env.single_observation_space, env.single_action_space, cfg, [128, 128], False, rnn, True)
    if kind == "qmix":
        return M.QMixNetwork(*args, dict(embed_dim=32, hypernet_layers=2, hypernet_embed=32), "cuda", max_batch=B, max_episode_length=T)
    return M.QNetwork(*args, "cuda", max_batch=B, max_episode_length=T)


@pytest.mark.parametrize("kind,rnn", [("idqn", False), ("qmix", False), ("idqn", True)])
def test_dqn_two_handles_with_summed_grads_match_the_union_batch(kind, rnn):
    from codebase_b200.dqn.train import Collector
    from codebase_b200.lbf import TrajStore

    B = 32
    envs = [_env(0), _env(P)]
    torch.manual_seed(0)
    ranks = [_dqn(kind, B, rnn, envs[0]) for _ in range(2)]
    union = _dqn(kind, 2 * B, rnn, envs[0])
    for m in (ranks[1], union):
        _copy_params(m, ranks[0])
    rb = TrajStore(2 * P, envs[0].n_agents, T, envs[0].cfg.obs_dim, ranks[0].device)
    for r in range(2):   # rank r's episodes in slots [r * P, (r + 1) * P)
        Collector(envs[r], ranks[0], T).collect(rb, r * P, 1.0)
    g = torch.Generator().manual_seed(1)
    for _ in range(3):   # the third update syncs the target (interval 2)
        idx = [(r * P + torch.randperm(P, generator=g)[:B]).to(torch.int32).cuda() for r in range(2)]
        for r in range(2):
            ranks[r].update_grads(rb, idx[r])
        _sum_into(zip(*[m.exchanged_buffers() for m in ranks]))
        met = [m.update_apply().clone() for m in ranks]
        union.update_grads(rb, torch.cat(idx))
        want = union.update_apply()
        assert torch.equal(met[0], met[1])
        assert abs(float(met[0][0]) - float(want[0])) <= 1e-5 * max(1.0, abs(float(want[0])))
        assert float(met[0][4]) == float(want[4])   # global filled count
    for name in ("theta", "theta_tgt", "adam_m", "adam_v") + (("mix", "mix_tgt", "mix_m", "mix_v") if kind == "qmix" else ()):
        a, b = getattr(ranks[0], name), getattr(ranks[1], name)
        assert torch.equal(a, b), f"{name} differs between the ranks"
        if name in ("theta", "theta_tgt", "mix", "mix_tgt"):
            _close(a, getattr(union, name), name)


def test_dqn_update_n_allreduce_on_one_rank_matches_update_n():
    """The driver's two-call loop with an identity exchange takes update_n's replay indices."""
    from codebase_b200.dqn.train import Collector
    from codebase_b200.lbf import TrajStore

    B, env = 32, _env(0)
    torch.manual_seed(0)
    a, b = _dqn("idqn", B, False, env), _dqn("idqn", B, False, env)
    _copy_params(b, a)
    rb = TrajStore(P, env.n_agents, T, env.cfg.obs_dim, a.device)
    Collector(env, a, T).collect(rb, 0, 1.0)
    a.update_n(rb, B, P, 11, 5, 4)
    b.update_n_allreduce(rb, B, P, 11, 5, 4, lambda bufs: None)
    _close(a.theta, b.theta, "theta")


# ---- actor-critic ----------------------------------------------------------------------------------------------------------------------------
def _ac(ppo, env, max_envs, actor_rnn=False):
    from codebase_b200.ac import model as M

    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=0.5, n_steps=5, entropy_coef=0.001, value_loss_coef=0.5,
                                target_update_interval_or_tau=200, standardise_returns=False, num_epochs=3, ppo_clip=0.2)
    actor = types.SimpleNamespace(layers=[128, 128], parameter_sharing=False, use_rnn=actor_rnn, use_orthogonal_init=True)
    critic = types.SimpleNamespace(layers=[128, 128], parameter_sharing=False, use_rnn=False, use_orthogonal_init=True, centralised=False)
    cls = M.PPONetwork if ppo else M.A2CNetwork
    return cls(env.single_observation_space, env.single_action_space, cfg, actor, critic, "cuda", max_envs=max_envs, max_episode_length=T)


def _ac_batches(model, envs):
    from codebase_b200.ac.train import Collector
    from codebase_b200.lbf import TrajStore

    halves = []
    for env in envs:
        c = Collector(env, model, T)
        c.collect()
        halves.append(c.batch)
    union = TrajStore(len(envs) * P, envs[0].n_agents, T, envs[0].cfg.obs_dim, model.device)
    for k in ("obs", "act", "rew", "done", "filled"):
        getattr(union, k).copy_(torch.cat([getattr(h, k) for h in halves]))
    return halves, union


@pytest.mark.parametrize("ppo", [False, True], ids=["ia2c", "ippo"])
def test_ac_two_handles_with_summed_grads_match_the_union_batch(ppo):
    envs = [_env(0), _env(P)]
    torch.manual_seed(0)
    ranks = [_ac(ppo, envs[0], P) for _ in range(2)]
    union = _ac(ppo, envs[0], 2 * P)
    for m in (ranks[1], union):
        _copy_params(m, ranks[0])
    for it, step in enumerate((0, 3200)):   # step 0 syncs the target critic
        halves, ub = _ac_batches(ranks[0], envs)
        epochs = ranks[0].num_epochs if ppo else 1
        for e in range(epochs):
            for r in range(2):
                if ppo:
                    ranks[r].epoch_grads(halves[r], P, e)
                else:
                    ranks[r].update_grads(halves[r], P)
            _sum_into([(ranks[0].grad, ranks[1].grad)])
            met = [(m.epoch_apply(step, e) if ppo else m.update_apply(step)).clone() for m in ranks]
        want = union.update_from_store(ub, 2 * P, step)
        assert torch.equal(met[0], met[1])
        for k in (0, 2, 3):
            assert abs(float(met[0][k]) - float(want[k])) <= 1e-4 * max(1.0, abs(float(want[k]))), (it, k)
        assert float(met[0][4]) == float(want[4])
    for name in ("theta", "theta_tgt", "adam_m", "adam_v"):
        a, b = getattr(ranks[0], name), getattr(ranks[1], name)
        assert torch.equal(a, b), f"{name} differs between the ranks"
        if name in ("theta", "theta_tgt"):
            _close(a, getattr(union, name), name)


@pytest.mark.parametrize("actor_rnn", [False, True], ids=["mlp", "gru_actor"])
def test_ppo_split_equals_the_fused_update(actor_rnn):
    env = _env(0)
    torch.manual_seed(0)
    fused, split = _ac(True, env, P, actor_rnn), _ac(True, env, P, actor_rnn)
    _copy_params(split, fused)
    for step in (0, 1600, 3200):
        halves, _ = _ac_batches(fused, [env])
        b = halves[0]
        m_f = fused.update_from_store(b, P, step).clone()
        for e in range(split.num_epochs):
            split.epoch_grads(b, P, e)
            split.epoch_apply(step, e)
        assert torch.equal(m_f, split._metrics)
        for name in ("theta", "theta_tgt", "adam_m", "adam_v"):
            assert torch.equal(getattr(fused, name), getattr(split, name)), name


def test_ppo_epoch_calls_check_their_arguments():
    from codebase_b200 import _native as nat

    m = _ac(True, _env(0), P)
    with pytest.raises(nat.NativeError, match="marl_ppo_prepare first"):
        m.epoch_apply(0, 0)
    halves, _ = _ac_batches(m, [_env(0)])
    m.epoch_grads(halves[0], P, 0)
    with pytest.raises(nat.NativeError, match="out of range"):
        m.epoch_apply(0, m.num_epochs)
    with pytest.raises(NotImplementedError, match="epoch_grads"):
        m.update_grads(halves[0], P)


# ---- env shards ------------------------------------------------------------------------------------------------------------------------------
def test_env_shards_collect_the_two_halves_of_one_env_set():
    from codebase_b200.dqn.train import Collector
    from codebase_b200.lbf import TrajStore

    whole = _env(0, 2 * P)
    shards = [_env(0), _env(P)]
    torch.manual_seed(0)
    model = _dqn("idqn", 32, False, whole)
    rb_whole = TrajStore(2 * P, whole.n_agents, T, whole.cfg.obs_dim, model.device)
    rb_shards = TrajStore(2 * P, whole.n_agents, T, whole.cfg.obs_dim, model.device)
    for _ in range(2):   # the second collection starts from the first one's env state
        Collector(whole, model, T).collect(rb_whole, 0, 0.5)
        for r in range(2):
            Collector(shards[r], model, T).collect(rb_shards, r * P, 0.5)
        for k in ("obs", "act", "rew", "done", "filled"):
            assert torch.equal(getattr(rb_whole, k), getattr(rb_shards, k)), k


# ---- torchrun end to end ---------------------------------------------------------------------------------------------------------------------
WRAPPER = r'''
import hashlib, os, sys
sys.path.insert(0, {root!r})
from codebase_b200 import run
from codebase_b200.ac import train as ac_train
from codebase_b200.dqn import train as dqn_train
from codebase_b200.utils import loggers

seen, steps = [], [0, 0]   # the learner; (this rank's env steps, the global env steps the driver counted)
_watch = loggers.Logger.watch
def watch(self, model):
    seen.append(model)
    return _watch(self, model)
loggers.Logger.watch = watch
_dqn_steps, _ac_steps = dqn_train.iteration_env_steps, ac_train.iteration_env_steps
def dqn_steps(final_len, dp):
    steps[0] += int(final_len.sum().item())
    g = _dqn_steps(final_len, dp); steps[1] += g
    return g
def ac_steps(t, P, dp):
    steps[0] += int(t) * int(P)
    g = _ac_steps(t, P, dp); steps[1] += g
    return g
dqn_train.iteration_env_steps, ac_train.iteration_env_steps = dqn_steps, ac_steps
run.main(sys.argv[2:])
h = hashlib.sha256()
for name in ("theta", "theta_tgt", "mix", "mix_tgt"):
    t = getattr(seen[0], name, None)
    if t is not None:
        h.update(t.detach().cpu().numpy().tobytes())
with open(os.path.join(sys.argv[1], "hash%s.txt" % os.environ.get("RANK", "0")), "w") as f:
    f.write("%s %d %d" % (h.hexdigest(), steps[0], steps[1]))
'''


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _launch(tmp_path, nproc, args, torchrun=True, timeout=900):
    """Runs the training command (under torchrun when `torchrun`), waits for it and kills its whole process group on a timeout."""
    script = tmp_path / "train.py"
    script.write_text(WRAPPER.format(root=ROOT))
    hashes = tmp_path / "hashes"
    hashes.mkdir(exist_ok=True)
    cmd = [sys.executable]
    if torchrun:
        cmd += ["-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={nproc}", f"--master-port={_free_port()}"]
    cmd += [str(script), str(hashes)] + args
    env = dict(os.environ, PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    p = subprocess.Popen(cmd, cwd=str(tmp_path), env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, start_new_session=True)
    try:
        out, _ = p.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        os.killpg(p.pid, signal.SIGKILL)
        p.communicate()
        raise
    finally:
        if p.poll() is None:
            os.killpg(p.pid, signal.SIGKILL)
    assert p.returncode == 0, out.decode(errors="replace")[-4000:]
    return sorted(hashes.iterdir())


JOBS = {
    "idqn": ["+algorithm=idqn", f"env.name={LBF}", "env.time_limit=25", "env.parallel_envs=32", "algorithm.training_start=0", "algorithm.batch_size=32",
             "algorithm.buffer_size=256", "algorithm.updates_per_iteration=4", "algorithm.eval_episodes=8"],
    "qmix": ["+algorithm=qmix", f"env.name={LBF}", "env.time_limit=25", "env.parallel_envs=32", "algorithm.training_start=0", "algorithm.batch_size=32",
             "algorithm.buffer_size=256", "algorithm.updates_per_iteration=4", "algorithm.eval_episodes=8"],
    "idqn_rnn": ["+algorithm=idqn", f"env.name={LBF}", "env.time_limit=25", "env.parallel_envs=32", "algorithm.training_start=0", "algorithm.batch_size=32",
                 "algorithm.buffer_size=256", "algorithm.updates_per_iteration=4", "algorithm.eval_episodes=8", "algorithm.model.use_rnn=True"],
    "ia2c": ["+algorithm=ia2c", f"env.name={LBF}", "env.time_limit=25", "env.parallel_envs=32"],
    "ippo_rware": ["+algorithm=ippo", "env.name=rware:rware-tiny-4ag-v2", "env.time_limit=100", "env.parallel_envs=16"],
}
STEPS = {"idqn": (8000, 2000), "qmix": (8000, 2000), "idqn_rnn": (8000, 2000), "ia2c": (8000, 1600), "ippo_rware": (16000, 3200)}   # (total, interval)


def _job(name, out):
    total, interval = STEPS[name]
    return JOBS[name] + ["seed=3", f"algorithm.total_steps={total}", f"algorithm.eval_interval={interval}", f"algorithm.save_interval={interval}", f"run_dir={out}"]


@pytest.mark.parametrize("name", sorted(JOBS))
def test_torchrun_two_ranks_on_one_device(tmp_path, name):
    import pandas as pd

    out = tmp_path / "out"
    hashes = _launch(tmp_path, 2, _job(name, out))
    assert [h.name for h in hashes] == ["hash0.txt", "hash1.txt"]
    (h0, local0, global0), (h1, local1, global1) = [h.read_text().split() for h in hashes]
    assert h0 == h1, "the ranks' parameters differ"
    # environment_steps counts the env steps of both ranks, and both ranks counted the same
    assert global0 == global1 and int(global0) == int(local0) + int(local1) and int(local0) > 0 and int(local1) > 0
    assert sorted(os.listdir(out)) == ["checkpoints", "config.yaml", "results.csv", "run.log"]
    assert not (tmp_path / "outputs").exists()
    df = pd.read_csv(out / "results.csv")
    total, interval = STEPS[name]
    steps = df["environment_steps"].to_numpy()
    assert len(df) >= 2 and (np.diff(steps) >= interval).all() and steps[-1] <= int(global0)
    assert len(os.listdir(out / "checkpoints")) >= 1
    assert np.isfinite(df["loss"].iloc[-1])


def test_torchrun_one_rank_reproduces_a_plain_run(tmp_path):
    import pandas as pd

    a, b = tmp_path / "a", tmp_path / "b"
    a.mkdir(); b.mkdir()
    ha = _launch(a, 1, _job("idqn", a / "out"), torchrun=False)
    hb = _launch(b, 1, _job("idqn", b / "out"), torchrun=True)
    assert ha[0].read_text() == hb[0].read_text()
    da, db = pd.read_csv(a / "out" / "results.csv"), pd.read_csv(b / "out" / "results.csv")
    cols = [c for c in da.columns if "episode_time" not in c]
    assert list(da.columns) == list(db.columns)
    pd.testing.assert_frame_equal(da[cols], db[cols])
    assert sorted(os.listdir(a / "out" / "checkpoints")) == sorted(os.listdir(b / "out" / "checkpoints"))
    for f in os.listdir(a / "out" / "checkpoints"):
        sa = torch.load(a / "out" / "checkpoints" / f, weights_only=True)
        sb = torch.load(b / "out" / "checkpoints" / f, weights_only=True)
        assert sa.keys() == sb.keys() and all(torch.equal(sa[k], sb[k]) for k in sa)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("name", ["idqn", "qmix", "ia2c"])
def test_torchrun_two_ranks_on_two_devices(tmp_path, name):
    out = tmp_path / "out"
    hashes = _launch(tmp_path, 2, _job(name, out))
    (h0, local0, global0), (h1, local1, global1) = [h.read_text().split() for h in hashes]
    assert h0 == h1, "the ranks' parameters differ"
    assert global0 == global1 and int(global0) == int(local0) + int(local1)
    assert sorted(os.listdir(out)) == ["checkpoints", "config.yaml", "results.csv", "run.log"]


# ---- the in-kernel peer exchange for QMIX and recurrent handles (two devices) ---------------------------------------------------------------------
def _peer_worker(rank, world, port, kind, out):
    import torch.distributed as dist

    from codebase_b200.dqn import model as M
    from codebase_b200.lbf import TrajStore

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    N, D, A, B = 2, 15, 6, 64
    space = types.SimpleNamespace
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=2, standardise_returns=False)
    rnn = kind == "idqn_rnn64"
    layers = [64, 64] if rnn else [128, 128]

    def make():
        torch.manual_seed(0)   # the same parameters on every rank
        args = ([space(shape=(D,), n=None)] * N, [space(shape=None, n=A)] * N, cfg, layers, False, rnn, True)
        if kind == "qmix":
            return M.QMixNetwork(*args, dict(embed_dim=32, hypernet_layers=2, hypernet_embed=32), f"cuda:{rank}", max_batch=B, max_episode_length=T)
        return M.QNetwork(*args, f"cuda:{rank}", max_batch=B, max_episode_length=T)

    rng = np.random.default_rng(100 + rank)   # different data per rank
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
    for k in range(3):   # the two-call form: update_grads, all-reduce of the agents' (and the mixer's) buffers, update_apply
        ref.update_grads(ts, idx[k])
        for buf in ref.exchanged_buffers():
            h = buf.cpu()
            dist.all_reduce(h)
            buf.copy_(h)
        ref.update_apply()
    torch.cuda.synchronize()
    names = ("theta", "theta_tgt") + (("mix", "mix_tgt") if kind == "qmix" else ())
    res = {"timed_out": peer.peer_timed_out()}
    for name in names:
        t = getattr(peer, name).cpu()
        gathered = [torch.empty_like(t) for _ in range(world)]
        dist.all_gather(gathered, t)
        res[name] = (all(torch.equal(gathered[0], g) for g in gathered), float((t - getattr(ref, name).cpu()).abs().max()))
    out.put((rank, res))
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs on one node")
@pytest.mark.parametrize("kind", ["qmix", "idqn_rnn64"])
def test_peer_exchange_covers_qmix_and_recurrent_handles(kind):
    """The mixer's gradient (QMIX) and a GRU handle that fits one wave ([64, 64]) in the in-kernel exchange: bit-identical across ranks and
    equal to the all-reduce form within 1e-6."""
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_peer_worker, args=(r, 2, port, kind, out)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=240)
    hung = [p for p in procs if p.is_alive()]
    for p in hung:
        p.kill()
    assert not hung, "a rank did not finish"
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    for rank, res in [out.get(timeout=10) for _ in range(2)]:
        assert not res.pop("timed_out"), f"rank {rank}: the in-kernel exchange gave up waiting for a peer"
        for name, (same, diff) in res.items():
            assert same, f"rank {rank}: {name} differs across ranks"
            assert diff <= 1e-6, (rank, name, diff)


def _attach_worker(rank, world, port, out):
    import torch.distributed as dist

    from codebase_b200 import _native as nat
    from codebase_b200.dqn import model as M

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(0)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    space = types.SimpleNamespace
    cfg = types.SimpleNamespace(optimizer="Adam", lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=2, standardise_returns=False)
    # rank 0: an MLP whose parameters fit the fused tail; rank 1: a GRU at [128, 128] (about 204 k parameters) that marl_dqn_peer_attach refuses
    m = M.QNetwork([space(shape=(15,), n=None)] * 2, [space(shape=None, n=6)] * 2, cfg, [128, 128], False, rank == 1, True, "cuda:0", max_batch=32,
                   max_episode_length=T)
    try:
        m.attach_peers()
        res = "attached"
    except nat.NativeError as e:
        res = str(e)
    dist.barrier()   # both ranks come back from attach_peers and reach the next collective
    out.put((rank, res))
    dist.destroy_process_group()


def test_attach_peers_fails_on_every_rank_when_one_rank_is_refused():
    """No update runs here (two ranks share this device): only the agreement on the outcome of attach_peers."""
    import torch.multiprocessing as mp

    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_attach_worker, args=(r, 2, port, out)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(timeout=240)
    hung = [p for p in procs if p.is_alive()]
    for p in hung:
        p.kill()
    assert not hung, "a rank did not come back from attach_peers"
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    res = dict(out.get(timeout=10) for _ in range(2))
    for rank in (0, 1):
        assert "peer-memory gradient exchange unavailable" in res[rank] and "rank 1:" in res[rank] and "do not fit" in res[rank], res

"""The reference's IDQN training loop restated on the CPU: marlbase/dqn/train.py:298-311 (collect one episode with one
env -> one sampled update), marlbase/dqn/model.py:94-116 (act: per-agent forward on a (1,1,obs) tensor, one
`random.random()` exploration test per step), 1 torch thread as marlbase/run.py:29 mandates.

TEST / MEASUREMENT INFRASTRUCTURE ONLY: this is what bench.py times as `cpu_baseline` and as `--impl reference`
(kind "port": the reference project and the third-party `lbforaging` package are not dependencies of this one).  The env is the
pure-Python restatement (oracle/lbf_ref.py), which has the same cost structure as upstream lbforaging (Python objects +
small numpy arrays); the learner is oracle/learner_ref.py (PyTorch CPU autograd + the Adam arithmetic of torch.optim).
"""
from __future__ import annotations

import random
import time

import numpy as np
import torch

from . import learner_ref as lr
from .lbf_ref import LBFConfig, WrappedForaging


class CpuIdqn:
    def __init__(self, cfg: LBFConfig, batch_size: int, buffer_size: int = 10000, seed: int = 0, hp: lr.DqnHP | None = None):
        torch.set_num_threads(1)  # run.py:29
        torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
        self.cfg, self.B, self.hp = cfg, batch_size, hp or lr.DqnHP()
        self.env = WrappedForaging(cfg, seed)
        self.N, self.D, self.A, self.T = cfg.n_agents, cfg.obs_dim, 6, cfg.time_limit
        theta = lr.init_flat(self.N, self.D, self.A)
        self.st = lr.DqnState(theta, theta.clone(), list(range(self.N)), self.D, self.A)
        self.rb = lr.ReplayRef(buffer_size, self.N, self.T, self.D)
        self.P = lr.net_size(self.D, self.A)

    def act(self, obss, epsilon):
        with torch.no_grad():  # the reference runs the forward even when it then explores (dqn/model.py:95-99,105)
            inputs = [torch.tensor(o).view(1, 1, -1) for o in obss]
            values = lr.agents_forward(self.st.theta, self.st.agent_net, inputs, self.D, self.A)
        if epsilon > random.random():
            return [random.randrange(self.A) for _ in range(self.N)]
        return [v.argmax(-1).squeeze().item() for v in values]

    def collect_episode(self, epsilon, use_network=True):
        obss, _ = self.env.reset()
        self.rb.init_episode(obss)
        done, t = False, 0
        while not done:
            actions = self.act(obss, epsilon) if use_network else [random.randrange(self.A) for _ in range(self.N)]
            obss, rews, d, trunc, _ = self.env.step(actions)
            done = d or trunc
            self.rb.add(obss, actions, rews, done)
            t += 1
        return t

    def update(self):
        idx = np.random.randint(0, len(self.rb), size=self.B)  # dqn/train.py:95
        return lr.dqn_update(self.st, lr.batch_from_store(self.rb.store, idx), self.hp)["loss"]

    def prefill(self, n_episodes):
        for _ in range(n_episodes):
            self.collect_episode(1.0, use_network=False)

    def run(self, n_episodes, epsilon=0.5):
        """n_episodes iterations of `collect one episode; one update` -> (env_steps, seconds)."""
        steps, t0 = 0, time.perf_counter()
        for _ in range(n_episodes):
            steps += self.collect_episode(epsilon)
            self.update()
        return steps, time.perf_counter() - t0


class CpuIa2c:
    """marlbase/ac/train.py:170-204 with ia2c.yaml's shape: P (default 10) envs stepped in lock-step until every env's first episode has
    ended (ac/train.py:24-119; the reference's AsyncVectorEnv subprocesses only parallelise env.step), then one A2CNetwork.update."""

    def __init__(self, cfg: LBFConfig, parallel_envs: int = 10, seed: int = 0, sharing: bool = True, hp: lr.A2CHP | None = None):
        torch.set_num_threads(1)
        torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
        self.cfg, self.P, self.hp = cfg, parallel_envs, hp or lr.A2CHP()
        self.envs = [WrappedForaging(cfg, seed, env_gid=i) for i in range(parallel_envs)]
        self.N, self.D, self.A, self.T = cfg.n_agents, cfg.obs_dim, 6, cfg.time_limit
        nets = [0] * self.N if sharing else list(range(self.N))
        n_nets = max(nets) + 1
        critic = lr.init_flat(n_nets, self.D, 1)
        self.st = lr.A2CState(lr.init_flat(n_nets, self.D, self.A), critic, critic.clone(), nets, nets, self.D, self.A)
        self.step = 0

    def iterate(self):
        P, N, T, D = self.P, self.N, self.T, self.D
        obs = np.zeros((T + 1, P, N * D), np.float32); act = np.zeros((T, P, N), np.int64); rew = np.zeros((T, P, N), np.float32)
        done = np.zeros((T + 1, P), np.float32); filled = np.zeros((T, P), np.float32)
        cur = [e.reset()[0] for e in self.envs]
        obs[0] = np.stack([np.concatenate(o) for o in cur])
        running, t, steps = np.ones(P, bool), 0, 0
        while running.any():
            with torch.no_grad():   # model.act on the whole vector (ac/model.py:147-153)
                xs = [torch.tensor(np.stack([cur[e][i] for e in range(P)])) for i in range(N)]
                logits = lr.agents_forward(self.st.actor, self.st.actor_net, xs, D, self.A)
                a = torch.stack([torch.distributions.Categorical(logits=l).sample() for l in logits], 1).numpy()
            for e in range(P):
                o, r, d, tr, _ = self.envs[e].step(a[e].tolist())
                if d or tr:
                    o = self.envs[e].reset()[0]   # vector-env autoreset
                cur[e] = o
                if running[e]:
                    obs[t + 1, e] = np.concatenate(o); act[t, e] = a[e]; rew[t, e] = r; done[t + 1, e] = float(d or tr); filled[t, e] = 1
                    steps += 1
                    if d or tr:
                        running[e] = False
            t += 1
        batch = dict(obss=torch.tensor(obs), actions=torch.tensor(act), rewards=torch.tensor(rew), dones=torch.tensor(done), filled=torch.tensor(filled))
        lr.a2c_update(self.st, batch, self.hp, self.step)
        self.step += t * P
        return steps

    def run(self, n_iterations, epsilon=None):
        steps, t0 = 0, time.perf_counter()
        for _ in range(n_iterations):
            steps += self.iterate()
        return steps, time.perf_counter() - t0

    def prefill(self, n):
        pass


def make_loop(algo, lbf, time_limit, batch, seed=0):
    """The CPU loop of one bench workload: 'idqn' | 'vdn' (CooperativeReward + agent-summed TD, vdn.yaml) | 'ia2c'."""
    cfg = LBFConfig(time_limit=time_limit, **lbf)
    if algo == "ia2c":
        return CpuIa2c(cfg, 10, seed=seed)
    return CpuIdqn(cfg, batch, seed=seed, hp=lr.DqnHP(mixer=int(algo == "vdn")))


def _pool_worker(conn, spec, seed):
    loop = make_loop(spec["algo"], spec["lbf"], spec["time_limit"], spec["batch"], seed=seed)
    loop.prefill(spec.get("prefill", 0))
    loop.run(1)
    conn.send("ready")
    while True:
        msg = conn.recv()
        if msg is None:
            return
        conn.send(loop.run(msg))


class WorkerPool:
    """`n_procs` persistent single-thread copies of the reference loop.  run_round(k): every copy runs k iterations; returns (env steps of all copies,
    wall-clock seconds of the round measured by the parent around the whole pool = the slowest copy)."""

    def __init__(self, n_procs, spec):
        import multiprocessing as mp

        ctx = mp.get_context("fork")
        self.conns, self.procs = [], []
        for i in range(n_procs):
            a, b = ctx.Pipe()
            p = ctx.Process(target=_pool_worker, args=(b, spec, 1000 + i), daemon=True)
            p.start()
            self.conns.append(a); self.procs.append(p)
        for c in self.conns:
            assert c.recv() == "ready"

    def run_round(self, k):
        t0 = time.perf_counter()
        for c in self.conns:
            c.send(k)
        res = [c.recv() for c in self.conns]
        return sum(r[0] for r in res), time.perf_counter() - t0

    def close(self):
        for c in self.conns:
            c.send(None)
        for p in self.procs:
            p.join(timeout=10)


def _worker(args):
    cfg_kw, batch_size, seed, prefill, n_episodes, n_rounds = args
    loop = CpuIdqn(LBFConfig(**cfg_kw), batch_size, seed=seed)
    loop.prefill(prefill)
    out = []
    for _ in range(n_rounds):
        out.append(loop.run(n_episodes))
    return out


def run_parallel(cfg_kw, batch_size, n_procs, prefill, n_episodes, n_rounds, pool=None):
    """`n_procs` independent single-thread copies of the reference loop (one per host core); returns per-round
    (total env steps, max seconds over workers, sum of per-copy rates)."""
    import multiprocessing as mp

    ctx = mp.get_context("fork")
    with ctx.Pool(n_procs) as p:
        res = p.map(_worker, [(cfg_kw, batch_size, 1000 + i, prefill, n_episodes, n_rounds) for i in range(n_procs)])
    rounds = []
    for r in range(n_rounds):  # (total env steps, slowest copy's seconds, sum of the copies' own steps/s)
        rounds.append((sum(w[r][0] for w in res), max(w[r][1] for w in res), sum(w[r][0] / w[r][1] for w in res)))
    return rounds

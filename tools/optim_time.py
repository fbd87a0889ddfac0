"""Per-update time of each optimiser (algorithm.optimizer) on BASELINE configs[1] -- IDQN on Foraging-8x8-2p-3f (2 agents x 15 features, T = 25),
batch 1024 from a 4096-episode replay ring, marl_dqn_update_n -- and on MAPPO (2 agents, centralised critic, 4096 envs, 4 epochs), plus the CUDA-event
time of the fused reduce + step tail of the IDQN update.  All five optimisers run in one call, alternating round by round after a warm-up, each
timed window about half a second (2 000 IDQN updates, 40 MAPPO updates); the card's name and power limit are read in the same call.  The tail's
kernel time comes from the profiler in a run of its own (`--tail`), so that tracing never overlaps the end-to-end windows.
Prints one JSON line:  python tools/optim_time.py [--tail]"""
import json
import os
import statistics
import sys
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import gpu_info  # noqa: E402
from codebase_b200.ac import model as AM  # noqa: E402
from codebase_b200.dqn import model as DM  # noqa: E402
from codebase_b200.lbf import TrajStore  # noqa: E402
from codebase_b200.optimizers import SUPPORTED  # noqa: E402

N, D, A, T = 2, 15, 6, 25
CAP, BATCH, ENVS, EPOCHS = 4096, 1024, 4096, 4
DQN_UPDATES, AC_UPDATES, ROUNDS = 2000, 40, 7


def sp(**kw):
    return types.SimpleNamespace(shape=kw.get("shape"), n=kw.get("n"))


def dqn(opt):
    cfg = types.SimpleNamespace(optimizer=opt, lr=3e-4, gamma=0.99, grad_clip=1.0, double_q=True, target_update_interval_or_tau=200, standardise_returns=False)
    return DM.QNetwork([sp(shape=(D,))] * N, [sp(n=A)] * N, cfg, [128, 128], False, False, True, "cuda", max_batch=BATCH, max_episode_length=T)


def mappo(opt):
    cfg = types.SimpleNamespace(optimizer=opt, lr=3e-4, gamma=0.99, grad_clip=0.5, n_steps=5, entropy_coef=0.001, value_loss_coef=0.5,
                                target_update_interval_or_tau=200, standardise_returns=False, num_epochs=EPOCHS, ppo_clip=0.2)
    net = types.SimpleNamespace(layers=[128, 128], parameter_sharing=False, use_rnn=False, use_orthogonal_init=True, centralised=False)
    cnet = types.SimpleNamespace(**{**vars(net), "centralised": True})
    return AM.PPONetwork([sp(shape=(D,))] * N, [sp(n=A)] * N, cfg, net, cnet, "cuda", max_envs=ENVS, max_episode_length=T)


def store(cap, device):
    ts = TrajStore(cap, N, T, D, device)
    ts.obs.copy_(torch.randint(-1, 9, ts.obs.shape, device=device).float()); ts.act.copy_(torch.randint(0, A, ts.act.shape))
    ts.rew.copy_((torch.rand_like(ts.rew) < 0.2).float()); ts.filled.fill_(1); ts.done[:, T] = 1
    return ts


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); fn(); b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def tail_us(m, ts):
    """mean CUDA time of the fused tail kernel (reduce_adam_kernel<0, OPT>) over 20 updates, from the profiler's kernel records"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        m.update_n(ts, BATCH, CAP, 7, 10_000, 20)
        torch.cuda.synchronize()
    times = [e.device_time for e in prof.events() if "reduce_adam_kernel" in e.name]
    return statistics.mean(times) if times else None


def main_tail():
    """profiler run: mean CUDA time of the fused tail kernel per optimiser (after a warm-up)"""
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    ts = store(CAP, dev)
    dq = {o: dqn(o) for o in SUPPORTED}
    for o in SUPPORTED:
        dq[o].update_n(ts, BATCH, CAP, 1, 0, 50)
    torch.cuda.synchronize()
    print(json.dumps({"gpu": gpu_info(torch, dev), "fused_tail_us": {o: tail_us(dq[o], ts) for o in SUPPORTED}}))
    for m in dq.values():
        m.close()


def main():
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    ts_dqn, ts_ac = store(CAP, dev), store(ENVS, dev)
    dq = {o: dqn(o) for o in SUPPORTED}
    ac = {o: mappo(o) for o in SUPPORTED}
    for o in SUPPORTED:   # warm-up: every shape of the timed window, once per optimiser
        dq[o].update_n(ts_dqn, BATCH, CAP, 1, 0, 10)
        for s in range(2):
            ac[o].update_from_store(ts_ac, ENVS, s)
    torch.cuda.synchronize()
    t_dqn = {o: [] for o in SUPPORTED}
    t_ac = {o: [] for o in SUPPORTED}
    first = 100
    for r in range(ROUNDS):   # alternate the optimisers round by round
        order = SUPPORTED[r % len(SUPPORTED):] + SUPPORTED[: r % len(SUPPORTED)]
        for o in order:
            t_dqn[o].append(1e3 * timed(lambda: dq[o].update_n(ts_dqn, BATCH, CAP, 1, first, DQN_UPDATES)) / DQN_UPDATES)
            t_ac[o].append(1e3 * timed(lambda: [ac[o].update_from_store(ts_ac, ENVS, s) for s in range(AC_UPDATES)]) / AC_UPDATES)
        first += DQN_UPDATES
    out = {"gpu": gpu_info(torch, dev), "idqn_us_per_update": {}, "mappo_us_per_update": {},
           "shape": dict(idqn=dict(agents=N, obs=D, T=T, batch=BATCH, replay=CAP), mappo=dict(agents=N, obs=D, T=T, envs=ENVS, epochs=EPOCHS)),
           "rounds": ROUNDS}
    for o in SUPPORTED:
        for key, t in (("idqn_us_per_update", t_dqn[o]), ("mappo_us_per_update", t_ac[o])):
            out[key][o] = dict(median=round(statistics.median(t), 2), min=round(min(t), 2), max=round(max(t), 2))
    print(json.dumps(out))
    for m in list(dq.values()) + list(ac.values()):
        m.close()


if __name__ == "__main__":
    main_tail() if "--tail" in sys.argv else main()

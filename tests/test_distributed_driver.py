"""CPU, world size 2 over gloo: the data-parallel plumbing of the training drivers (codebase_b200/distributed.py, run.py, dqn/train.py,
ac/train.py) -- run-directory broadcast and rank-0-only writes, the global env-step arithmetic of both drivers, env-id sharding, the collectives'
bit-identical results, and what stays refused on several ranks.  No GPU, no product kernels."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from codebase_b200 import distributed
from codebase_b200.config import compose

ARGS = ["+algorithm=idqn", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "seed=0"]


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _environ(rank, world, port):
    return {"RANK": str(rank), "WORLD_SIZE": str(world), "LOCAL_RANK": str(rank), "LOCAL_WORLD_SIZE": str(world),
            "MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port)}


def _worker(rank, world, port, base, out):
    os.environ.update(_environ(rank, world, port))
    torch.set_num_threads(1)
    from codebase_b200 import run
    from codebase_b200.ac import train as ac_train
    from codebase_b200.dqn import train as dqn_train
    from codebase_b200.utils.loggers import NullLogger

    cfg = compose(ARGS)
    dp = distributed.init(cfg)
    try:
        assert distributed.current() is dp and dp.active and dp.backend == "gloo" and dp.rank == rank
        # run directory: chosen by rank 0 (random hex), the same on every rank; only rank 0's logger writes
        os.chdir(base)
        logger = run.enter_run_dir(cfg, dp)
        out[f"cwd{rank}"] = os.getcwd()
        out[f"null{rank}"] = isinstance(logger, NullLogger)
        dp.gather_objects(None)   # rank 0 has written config.yaml before any rank logs
        logger.log_metrics([{"episode_returns": float(rank), "episode_length": 25}, {"episode_returns": float(rank) + 1, "episode_length": 20},
                            {"updates": 1, "environment_steps": 100}])
        # the drivers' global step: DQN sums every episode length, actor-critic sums t x P of every rank
        final_len = torch.tensor([3, 25, 7] if rank == 0 else [25, 1], dtype=torch.int32)
        out[f"dqn_steps{rank}"] = dqn_train.iteration_env_steps(final_len, dp)
        out[f"ac_steps{rank}"] = ac_train.iteration_env_steps(int(final_len.max()), 4 + rank, dp)
        # collectives: the sum of several buffers in one exchange, bit-identical on every rank; broadcast from rank 0
        g = torch.Generator().manual_seed(rank)
        a, b = torch.randn(1000, generator=g), torch.randn(37, generator=g)
        out[f"parts{rank}"] = (a.clone(), b.clone())
        dp.all_reduce_([a, b])
        out[f"sum{rank}"] = (a, b)
        c = torch.full((5,), float(rank + 1))
        dp.broadcast_(c)
        out[f"bcast{rank}"] = c
        out[f"shard{rank}"] = distributed.shard(rank, 8)
        dp.gather_objects(None)
    finally:
        distributed.finish()


def test_two_ranks_share_one_run_dir_and_only_rank_0_writes(tmp_path):
    base = tmp_path / "base"
    base.mkdir()
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(2, _free_port(), str(base), out), nprocs=2, join=True)
    # run directory
    assert out["cwd0"] == out["cwd1"] and out["cwd0"].startswith(str(base / "outputs"))
    assert not out["null0"] and out["null1"]
    run_dir = out["cwd0"]
    assert sorted(os.listdir(run_dir)) == ["config.yaml", "results.csv", "run.log"]
    import pandas as pd

    df = pd.read_csv(os.path.join(run_dir, "results.csv"))
    assert len(df) == 1 and df["mean_episode_returns"].iloc[0] == 0.5    # rank 0's line only
    assert len(list((base / "outputs").rglob("*"))) == 6                # outputs/<env>/<algorithm>/<hex>/ + its three files
    # global env steps: (3 + 25 + 7) + (25 + 1); actor-critic 25 x 4 + 25 x 5
    assert out["dqn_steps0"] == out["dqn_steps1"] == 61
    assert out["ac_steps0"] == out["ac_steps1"] == 25 * 4 + 25 * 5
    # collectives
    a0, b0 = out["parts0"]
    a1, b1 = out["parts1"]
    for r in (0, 1):
        a, b = out[f"sum{r}"]
        assert torch.equal(a, a0 + a1) and torch.equal(b, b0 + b1)
        assert torch.equal(out[f"bcast{r}"], torch.full((5,), 1.0))
    # env-id sharding: rank r owns [r * P, (r + 1) * P)
    assert (out["shard0"], out["shard1"]) == (0, 8)


def test_shards_reproduce_the_unsharded_envs():
    """The global env ids of two shards are those of one env set twice the size: the same boards after reset."""
    from oracle import lbf_c

    P = 8
    shards = [lbf_c.OracleVecEnv(lbf_c.make_cfg(), P, seed=5, env_gid0=distributed.shard(r, P)).reset() for r in range(2)]
    whole = lbf_c.OracleVecEnv(lbf_c.make_cfg(), 2 * P, seed=5, env_gid0=0).reset()
    assert np.array_equal(np.concatenate(shards), whole)


def test_single_process_starts_no_group():
    cfg = compose(ARGS)
    for env in ({}, {"WORLD_SIZE": "1", "RANK": "0", "LOCAL_RANK": "0"}):
        dp = distributed.init(cfg, environ=env)
        assert not dp.active and dp.rank == 0 and dp.world == 1 and dp.is_main
        assert dp.sum_int(7) == 7 and dp.gather_objects("x") == ["x"] and dp.broadcast_object(3) == 3
        t = torch.ones(3)
        dp.all_reduce_([t])
        assert torch.equal(t, torch.ones(3))
        distributed.finish()
    assert not torch.distributed.is_initialized()


@pytest.mark.parametrize("alg", ["idqn", "ia2c", "ippo", "qmix"])
def test_standardise_returns_is_refused_on_several_ranks(alg):
    cfg = compose([f"+algorithm={alg}", "env.name=lbforaging:Foraging-8x8-2p-3f-v3", "env.time_limit=25", "algorithm.standardise_returns=True"])
    with pytest.raises(NotImplementedError, match="standardise_returns"):
        distributed.init(cfg, environ=_environ(0, 2, 1))
    assert not torch.distributed.is_initialized()
    dp = distributed.init(cfg, environ=_environ(0, 1, 1))   # one rank: allowed
    assert not dp.active


def test_unsupported_worlds_are_refused():
    cfg = compose(ARGS)
    with pytest.raises(NotImplementedError, match="at most 8 ranks"):
        distributed.init(cfg, environ=_environ(0, 9, 1))
    env = _environ(0, 4, 1)
    env["LOCAL_WORLD_SIZE"] = "2"
    with pytest.raises(NotImplementedError, match="one node"):
        distributed.init(cfg, environ=env)
    assert not torch.distributed.is_initialized()


def test_backend_choice():
    """From the ranks' device UUIDs: one visible device per process (device_count() == 1 everywhere) still means a device per rank."""
    assert distributed.choose_backend(["GPU-a", "GPU-b"]) == "nccl"
    assert distributed.choose_backend(["GPU-a", "GPU-a"]) == "gloo" and distributed.choose_backend(["GPU-a", "GPU-b", "GPU-a"]) == "gloo"
    assert distributed.choose_backend([None, None]) == "gloo"

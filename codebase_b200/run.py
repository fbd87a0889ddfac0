"""Entry point -- drop-in for marlbase/run.py:14-47 with the same command line:

    python -m codebase_b200.run +algorithm=idqn env.name="lbforaging:Foraging-8x8-2p-3f-v3" env.time_limit=25 seed=0

Builds logger, env, a second evaluation env, seeds torch/numpy, dispatches `algorithm._target_`, and works in
outputs/<env.name>/<algorithm.name>/<random hex>/ (results.csv, config.yaml) exactly as the reference's Hydra run dir
(configs/default.yaml:7-9).

Data-parallel training on several GPUs of one node (weak scaling, codebase_b200/distributed.py):

    torchrun --nproc-per-node 2 -m codebase_b200.run +algorithm=idqn env.name="lbforaging:Foraging-8x8-2p-3f-v3" env.time_limit=25 seed=0

Rank 0 chooses the run directory and alone writes config.yaml, results.csv, run.log and checkpoints/; rank r collects env.parallel_envs envs
with global ids [r * P, (r + 1) * P); only rank 0 evaluates."""
from __future__ import annotations

import logging
import os
import sys

import numpy as np
import torch

from . import distributed
from .config import Config, call, compose, instantiate
from .utils.loggers import NullLogger


def main(argv=None):
    cfg = compose(list(sys.argv[1:] if argv is None else argv))
    dp = distributed.init(cfg)
    try:
        return _run(cfg, dp)
    finally:
        distributed.finish()


def enter_run_dir(cfg, dp):
    """Rank 0 chooses (and creates) the run directory and broadcasts it; every rank works in it.  Returns the logger: rank 0's writes
    config.yaml, results.csv and run.log, the other ranks' writes nothing."""
    run_dir = None
    if dp.is_main:
        run_dir = cfg.get("run_dir") or os.path.join("outputs", str(cfg.env.name), str(cfg.algorithm.get("name", "algorithm")), os.urandom(4).hex())
        os.makedirs(run_dir, exist_ok=True)
    run_dir = dp.broadcast_object(run_dir)
    os.chdir(run_dir)
    if dp.is_main:
        logging.basicConfig(level=logging.INFO, format="[%(asctime)s][%(levelname)s] - %(message)s",
                            handlers=[logging.FileHandler("run.log"), logging.StreamHandler(sys.stdout)], force=True)
        return instantiate(cfg.logger, cfg=cfg)
    # warnings and errors of the other ranks still reach stderr
    logging.basicConfig(level=logging.WARNING, format=f"[rank {dp.rank}][%(levelname)s] - %(message)s", handlers=[logging.StreamHandler(sys.stderr)], force=True)
    return NullLogger("", cfg)


def _run(cfg, dp):
    logger = enter_run_dir(cfg, dp)
    if dp.active:
        env = call(cfg.env, seed=cfg.seed, env_gid0=distributed.shard(dp.rank, cfg.env.get("parallel_envs") or 1))
    else:
        env = call(cfg.env, seed=cfg.seed)
    # evaluation envs: the reference builds ONE extra env (run.py:21-27); here `eval_episodes` instances run one episode each (rank 0 only)
    eval_env = None
    if dp.is_main:
        eval_cfg = Config(cfg.env.to_dict())
        eval_cfg["parallel_envs"] = int(cfg.algorithm.eval_episodes)
        eval_env = call(eval_cfg, seed=cfg.seed, env_gid0=1 << 30)
    torch.set_num_threads(1)
    if cfg.seed is not None:
        torch.manual_seed(cfg.seed)
        np.random.seed(cfg.seed)
    else:
        logger.warning("No seed has been set.")
    assert cfg.env.time_limit is not None, "Time limit must be set."
    algo = cfg.algorithm
    algo["seed_for_sampling"] = cfg.seed
    call(algo, env, eval_env, logger, time_limit=cfg.env.time_limit)
    return logger.get_state()


if __name__ == "__main__":
    main()

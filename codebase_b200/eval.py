"""Evaluate a checkpoint of a finished (or running) run -- the role of marlbase/eval.py:16-64 with the same arguments:

    python -m codebase_b200.eval path=outputs/<env>/<alg>/<hex> [load_step=N] [seed=S] [episodes=K]

Like the reference it reads `<path>/config.yaml`, builds the run's env, picks `checkpoints/model_s<load_step>.pt` (the latest when load_step is
not given), swaps `algorithm._target_`'s "train" for "eval" and calls it with (env, ckpt_path, **algorithm).  The reference's eval targets record
a video of `video_frames` steps (dqn/eval.py, ac/eval.py); rendering is out of scope of the GPU path, so ours run `episodes` evaluation episodes on
the device with the loaded parameters and write their returns to `<path>/eval_s<load_step>.json` instead."""
from __future__ import annotations

import os
import re
import sys

import numpy as np
import torch
import yaml

from .config import Config, call


def latest_step(ckpt_dir: str) -> int:
    """marlbase/eval.py:46-52: the largest N over checkpoints/model_sN.pt"""
    steps = [int(m.group(1)) for f in os.listdir(ckpt_dir) if (m := re.fullmatch(r"model_s(\d+)\.pt", f))]
    if not steps:
        raise FileNotFoundError(f"no model_s*.pt under {ckpt_dir}")
    return max(steps)


def parse_args(argv):
    out = dict(path=None, load_step=None, seed=None, episodes=None)
    for a in argv:
        k, sep, v = a.partition("=")
        if not sep or k not in out:
            raise ValueError(f"unknown argument {a!r}: expected path=... [load_step=N] [seed=S] [episodes=K]")
        out[k] = None if v in ("null", "None", "") else (v if k == "path" else int(v))
    return out


def main(argv=None):
    args = parse_args(list(sys.argv[1:] if argv is None else argv))
    path = args["path"]
    assert path and os.path.isdir(path), f"Path {path} is not a directory."
    config_path = os.path.join(path, "config.yaml")
    assert os.path.exists(config_path), f"Config file {config_path} does not exist."
    with open(config_path) as f:
        run_config = Config(yaml.safe_load(f))
    load_step = args["load_step"] if args["load_step"] is not None else latest_step(os.path.join(path, "checkpoints"))
    ckpt_path = os.path.join(path, "checkpoints", f"model_s{load_step}.pt")
    assert os.path.exists(ckpt_path), f"Checkpoint {ckpt_path} does not exist."
    seed = args["seed"] if args["seed"] is not None else run_config.get("seed")
    env_cfg = Config(run_config.env.to_dict())
    env_cfg["parallel_envs"] = int(args["episodes"] or run_config.algorithm.get("eval_episodes", 100))   # one episode per env instance
    env = call(env_cfg, seed=seed, env_gid0=1 << 29)
    torch.set_num_threads(1)
    if seed is not None:
        torch.manual_seed(seed)
        np.random.seed(seed)
    algo = Config(run_config.algorithm.to_dict())
    algo["_target_"] = str(algo["_target_"]).replace("train", "eval")
    result = call(algo, env, ckpt_path, time_limit=run_config.env.time_limit)
    result.update(load_step=int(load_step), checkpoint=os.path.abspath(ckpt_path))
    import json

    with open(os.path.join(path, f"eval_s{load_step}.json"), "w") as f:
        json.dump(result, f)
    print(f"step {load_step}: mean return {result['mean_episode_returns']:.4f} +- {result['std_episode_returns']:.4f} over {result['episodes']} episodes")
    return result


if __name__ == "__main__":
    main()

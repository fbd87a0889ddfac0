"""`ac.eval.main(env, ckpt_path, **cfg)` -- marlbase/ac/eval.py:8-27: load the checkpoint into the run's model class, sample one episode per env
instance from the policy (the reference's `model.act` samples from the categorical as well), and with `video_path` record `video_frames` frames
of the policy there (train.record_episodes)."""
from __future__ import annotations

import os

import torch

from ..config import Config, instantiate
from ..dqn.eval import summarise
from ..utils import video
from .train import Collector, record_episodes


def main(env, ckpt_path, time_limit, video_path=None, **cfg):
    cfg = Config(cfg)
    model = instantiate(cfg.model, env.single_observation_space, env.single_action_space, cfg, max_envs=env.num_envs, max_episode_length=time_limit)
    print(f"Loading model from {ckpt_path}")
    model.load_state_dict(torch.load(ckpt_path, weights_only=True))
    ln, ret = Collector(env, model, time_limit).collect()
    torch.cuda.synchronize()
    out = summarise(ln, ret)
    if video_path:
        venv = video.recording_env(env)
        record_episodes(venv, model, cfg.video_frames, video_path)
        venv.close()
        out["video"] = os.path.abspath(video_path)
    env.close()
    return out

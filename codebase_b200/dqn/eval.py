"""`dqn.eval.main(env, ckpt_path, **cfg)` -- marlbase/dqn/eval.py:8-28: instantiate the model from the run's config, load the checkpoint
(`torch.load(..., weights_only=True)` + `load_state_dict`, the reference's two lines), play one greedy-ish episode (`eps_evaluation`) per env
instance on the device, and with `video_path` record `video_frames` frames of the policy there (train.record_episodes)."""
from __future__ import annotations

import os

import torch

from ..config import Config, instantiate
from ..utils import video
from .train import Collector, record_episodes


def summarise(final_len, final_ret):
    ln, ret = final_len.cpu().numpy(), final_ret.cpu().numpy().sum(-1)   # the logged episode return is the sum over agents (utils/wrappers.py:33-41)
    return dict(episodes=int(len(ln)), mean_episode_returns=float(ret.mean()), std_episode_returns=float(ret.std()), mean_episode_length=float(ln.mean()),
                episode_returns=[float(x) for x in ret])


def main(env, ckpt_path, time_limit, video_path=None, **cfg):
    cfg = Config(cfg)
    model = instantiate(cfg.model, env.single_observation_space, env.single_action_space, cfg, max_batch=cfg.batch_size, max_episode_length=time_limit)
    print(f"Loading model from {ckpt_path}")
    model.load_state_dict(torch.load(ckpt_path, weights_only=True))
    ln, ret = Collector(env, model, time_limit).collect(None, 0, cfg.eps_evaluation)
    torch.cuda.synchronize()
    out = summarise(ln, ret)
    if video_path:
        venv = video.recording_env(env)
        record_episodes(venv, model, cfg.video_frames, video_path, cfg.eps_evaluation)
        venv.close()
        out["video"] = os.path.abspath(video_path)
    env.close()
    return out

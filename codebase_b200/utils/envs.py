"""Env factory on the GPU path -- drop-in for marlbase/utils/envs.py (`env._target_: utils.envs.make_env`,
configs/default.yaml:28-35).  Returns a vector env whose transition runs in libmarlb200.so (marl_lbf_*).

`B200VecEnv` speaks the gymnasium<1.0 vector protocol the reference's drivers rely on (marlbase/ac/train.py:30-34,
79-110): `single_observation_space`, `single_action_space`, `observation_space[0].shape[0] == parallel_envs`,
`reset() -> (tuple of N arrays [P, obs], info)`, `step(actions) -> (obs, rewards [P, N], done [P], truncated [P],
info)` with same-step autoreset and `info["final_info"][i]` carrying `episode_returns`, `agent{i}/episode_returns`,
`episode_length`, `episode_time` (marlbase/utils/wrappers.py:36-41).  Not provided: gymnasium's `info["final_observation"]` -- the transition kernel
resets a finished env in the same launch and only the first observation of the next episode leaves it; the reference's drivers never read that key
(ac/train.py:90-110 use `final_info` only).  The native drivers (dqn/train.py, ac/train.py
of this package) skip the numpy surface and drive `env.native` with device tensors.
"""
from __future__ import annotations

import random
from time import perf_counter

import numpy as np
import torch

from ..lbf import LbfConfig, NativeLbf, parse_env_id
from . import spaces

SUPPORTED_WRAPPERS = {"CooperativeReward"}


class _Unwrapped:
    def __init__(self, n_agents):
        self.n_agents = n_agents


class B200VecEnv:
    def __init__(self, cfg: LbfConfig, parallel_envs: int, seed: int, env_gid0: int = 0, device=None):
        self.cfg, self.num_envs = cfg, int(parallel_envs)
        self.native = NativeLbf(cfg, self.num_envs, seed, env_gid0, device)
        self.n_agents = cfg.n_agents
        self.unwrapped = _Unwrapped(cfg.n_agents)
        hi = float(max(cfg.rows, cfg.cols))
        self.single_observation_space = spaces.Tuple([spaces.Box(-1.0, hi, (cfg.obs_dim,), np.float32)] * cfg.n_agents)
        self.single_action_space = spaces.Tuple([spaces.Discrete(cfg.n_actions)] * cfg.n_agents)
        self.observation_space = spaces.Tuple([spaces.Box(-1.0, hi, (self.num_envs, cfg.obs_dim), np.float32)] * cfg.n_agents)
        self.action_space = spaces.Tuple([spaces.Discrete(cfg.n_actions)] * cfg.n_agents)
        self._t0 = perf_counter()

    # ---- gymnasium-style surface (numpy in / numpy out) ------------------------------------------------------------
    def _obs_tuple(self, obs):
        o = obs.cpu().numpy()
        return tuple(o[:, i] for i in range(self.n_agents))

    def reset(self, seed=None, options=None):
        self._t0 = perf_counter()
        return self._obs_tuple(self.native.reset()), {}

    def step(self, actions):
        """`actions`: the reference's layout only -- one sequence of `parallel_envs` actions per agent, i.e. [N][P]
        (`actions.squeeze().tolist()` of model.act's i64[N, P, 1], marlbase/ac/train.py:79-81); with one env also the flat
        per-agent list [N] of the single-env protocol (marlbase/dqn/train.py:217)."""
        a = np.asarray(actions)
        if a.ndim == 3 and a.shape[-1] == 1:
            a = a[..., 0]
        if a.shape == (self.n_agents,) and self.num_envs == 1:
            a = a[:, None]
        if a.shape != (self.n_agents, self.num_envs):
            raise ValueError(f"actions must have shape (n_agents={self.n_agents}, parallel_envs={self.num_envs}), got {a.shape}")
        a = torch.as_tensor(a.T.copy(), dtype=torch.int32, device=self.native.device).contiguous()
        obs, rew, done, trunc = self.native.step(a, autoreset=True)
        done_h, trunc_h = done.cpu().numpy().astype(bool), trunc.cpu().numpy().astype(bool)
        info = {}
        fin = done_h | trunc_h
        if fin.any():
            ret, ln = self.native.final_ret.cpu().numpy(), self.native.final_len.cpu().numpy()
            now = perf_counter()
            final = np.full(self.num_envs, None, dtype=object)
            for i in np.nonzero(fin)[0]:
                final[i] = episode_info(ret[i], int(ln[i]), now - self._t0)
            info["final_info"], info["_final_info"] = final, fin
        return self._obs_tuple(obs), rew.cpu().numpy(), done_h, trunc_h, info

    def close(self):
        self.native.close()


def episode_info(returns, length, seconds):
    """The keys RecordEpisodeStatistics adds at episode end (marlbase/utils/wrappers.py:36-41)."""
    info = {"episode_returns": np.asarray(returns, np.float32)}
    for i, r in enumerate(returns):
        info[f"agent{i}/episode_returns"] = np.float32(r)
    info["episode_length"] = int(length)
    info["episode_time"] = float(seconds)
    return info


def make_env(seed, enable_video=False, name=None, time_limit=None, clear_info=False, observe_id=False, standardise_rewards=False,
             wrappers=None, parallel_envs=None, env_gid0=0, device=None, **kwargs):
    """marlbase/utils/envs.py:115-119 with the same config keys.  `parallel_envs` absent -> 1 env (the reference's single-env
    factory); the GPU overlays set it to thousands."""
    if enable_video:
        raise NotImplementedError("video recording is out of scope of the GPU hot path (algorithm.video_interval must stay False)")
    wrappers = list(wrappers or [])
    unknown = [w for w in wrappers if w not in SUPPORTED_WRAPPERS]
    if unknown:
        raise NotImplementedError(f"env.wrappers {unknown} are not implemented on the GPU path (supported: {sorted(SUPPORTED_WRAPPERS)})")
    cfg = parse_env_id(name, time_limit or 0, **kwargs)
    cfg.cooperative_reward = int("CooperativeReward" in wrappers)
    cfg.observe_id, cfg.standardise_rewards = int(bool(observe_id)), int(bool(standardise_rewards))   # envs.py:97-101, inside the listed wrappers
    if seed is None:
        seed = random.randint(0, 99999)  # envs.py:58-59
    return B200VecEnv(cfg, int(parallel_envs or 1), int(seed), env_gid0, device)

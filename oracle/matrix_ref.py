"""CPU restatement of the repeated matrix games (``matrixgames`` ``MatrixGame``: climbing, penalty-k) under marlbase's wrapper stack --
numpy, one env per object.  TEST INFRASTRUCTURE ONLY: the CUDA kernel (codebase_b200/csrc/matrix_env.cu) is checked against it bit for bit.
PARITY UNPINNED against upstream ``matrixgames`` (absent from the reference checkout): the semantics are the ones DESIGN.md Appendix C
restates from memory.
"""
from __future__ import annotations

import numpy as np

from .lbf_ref import StandardiseReward


class MatrixGame:
    """MatrixGame(payoff_matrix, ep_length, last_action_state): N = payoff.ndim players, player i has payoff.shape[i] actions."""

    def __init__(self, payoff, ep_length=25, last_action_state=True):
        self.payoff = np.asarray(payoff)
        self.n_agents = self.payoff.ndim
        self.ep_length = int(ep_length)
        self.last_action_state = bool(last_action_state)
        self.t = 0
        self.last_actions = None   # None: no action since the reset

    def observation(self):
        if not self.last_action_state:
            return [np.zeros(1, np.float32) for _ in range(self.n_agents)]
        obs = np.zeros(sum(self.payoff.shape), np.float32)
        if self.last_actions is not None:
            off = 0
            for a, n in zip(self.last_actions, self.payoff.shape):
                obs[off + a] = 1.0
                off += n
        return [obs.copy() for _ in range(self.n_agents)]

    def reset(self):
        self.t = 0
        self.last_actions = None
        return self.observation()

    def step(self, actions):
        """Returns (obs, rewards: N copies of payoff[actions] in the table's dtype, terminated)."""
        actions = tuple(int(a) for a in actions)
        self.t += 1
        self.last_actions = actions
        r = self.payoff[actions]
        return self.observation(), [r] * self.n_agents, self.t >= self.ep_length


class WrappedMatrixGame:
    """MatrixGame under marlbase's wrapper stack: TimeLimit(time_limit) -> RecordEpisodeStatistics -> [ObserveID] -> [StandardiseReward] ->
    [CooperativeReward] (marlbase/utils/envs.py:93-109), the optional wrappers' arithmetic as oracle/lbf_ref.WrappedForaging has it.
    cfg: a codebase_b200.matrix.MatrixConfig (payoff, ep_length, last_action_state and the wrapper flags)."""

    def __init__(self, cfg, payoff=None):
        self.cfg = cfg
        self.env = MatrixGame(cfg.payoff if payoff is None else payoff, cfg.ep_length, cfg.last_action_state)
        self.n_resets = 0
        self.episode_reward = np.zeros(cfg.n_agents, np.float32)
        self.episode_length = 0
        self.stdr = StandardiseReward(cfg.n_agents)

    def observation(self, obs=None):
        obs = np.stack(self.env.observation() if obs is None else obs)
        if self.cfg.observe_id:
            obs = np.concatenate((np.eye(self.cfg.n_agents, dtype=obs.dtype), obs), axis=1)
        return obs

    def reset(self):
        self.n_resets += 1
        self.episode_reward = np.zeros(self.cfg.n_agents, np.float32)
        self.episode_length = 0
        return self.observation(self.env.reset())

    def step(self, actions):
        """Returns (obs [N][D], rewards float32 [N], terminated, truncated, info)."""
        c = self.cfg
        obs, reward, done = self.env.step(actions)
        truncated = bool(c.time_limit > 0 and self.env.t >= c.time_limit)
        info = {}
        self.episode_reward = self.episode_reward + np.array(reward, dtype=np.float32)
        self.episode_length += 1
        if done or truncated:
            info["episode_returns"] = self.episode_reward.copy()
            info["episode_length"] = self.episode_length
        if c.standardise_rewards:
            reward = self.stdr.reward(reward)
        if c.cooperative_reward:
            reward = c.n_agents * [sum(reward)]
        return self.observation(obs), np.asarray(reward, np.float32), done, truncated, info


class OracleVecMatrix:
    """E wrapped matrix games with the native handle's step semantics (autoreset in the same step, inactive envs after an ended episode).
    An action outside 0..A-1 is played as action 0, as the kernel does (upstream would index the table with it)."""

    def __init__(self, cfg, E):
        self.cfg, self.E, self.N, self.D, self.A = cfg, E, cfg.n_agents, cfg.obs_dim, cfg.n_actions
        self.envs = [WrappedMatrixGame(cfg) for _ in range(E)]
        self.active = np.ones(E, np.uint8)

    @property
    def episode_idx(self):
        return np.array([w.n_resets for w in self.envs], np.int64)

    @property
    def step_count(self):
        return np.array([w.env.t for w in self.envs], np.int64)

    def reset(self, mask=None):
        obs = np.zeros((self.E, self.N, self.D), np.float32)
        for e, w in enumerate(self.envs):
            if mask is None or mask[e]:
                w.reset()
                self.active[e] = 1
            obs[e] = w.observation()
        return obs

    def step(self, actions, autoreset=False):
        E, N = self.E, self.N
        obs = np.zeros((E, N, self.D), np.float32)
        rew = np.zeros((E, N), np.float32)
        done, trunc = np.ones(E, np.uint8), np.zeros(E, np.uint8)
        fret, flen = np.zeros((E, N), np.float32), np.zeros(E, np.int32)
        for e, w in enumerate(self.envs):
            if not self.active[e]:
                obs[e] = w.observation()
                continue
            a = [int(x) if 0 <= int(x) < self.A else 0 for x in actions[e]]
            o, r, d, t, info = w.step(a)
            rew[e], done[e], trunc[e] = r, d, t
            if d or t:
                fret[e], flen[e] = info["episode_returns"], info["episode_length"]
                if autoreset:
                    o = w.reset()
                else:
                    self.active[e] = 0
            obs[e] = o
        return obs, rew, done, trunc, fret, flen

    def load(self, last_action, step):
        """The kernel's set_state: previous actions int [E][N] (-1: none), step counts [E]; returns and lengths restart, envs become active."""
        for e, w in enumerate(self.envs):
            la = [int(x) for x in last_action[e]]
            w.env.last_actions = None if la[0] < 0 else tuple(la)
            w.env.t = int(step[e])
            w.episode_reward = np.zeros(self.N, np.float32)
            w.episode_length = 0
            w.n_resets = max(w.n_resets, 1)
        self.active[:] = 1

    def state(self):
        last = np.array([[-1] * self.N if w.env.last_actions is None else list(w.env.last_actions) for w in self.envs], np.int8)
        return dict(last_action=last, step=self.step_count.astype(np.int32),
                    ep_return=np.stack([w.episode_reward for w in self.envs]).astype(np.float32),
                    ep_len=np.array([w.episode_length for w in self.envs], np.int32), episode_idx=self.episode_idx.astype(np.int32),
                    active=self.active.copy())

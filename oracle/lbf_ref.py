"""Second, independent CPU restatement of lbforaging's ``ForagingEnv`` -- pure Python, one env, written
object-by-object the way the upstream package structures it (players, a numpy field, a collisions
dict, a loading set).  TEST INFRASTRUCTURE ONLY (see oracle/lbf_oracle.h): it exists so the C oracle
(``lbf_oracle.c``) is cross-checked by something that does not share its code, and as the readable
specification.  PARITY UNPINNED against upstream ``lbforaging`` (third-party, un-vendored, unpinned;
reference call sites marlbase/utils/envs.py:27-37,90-92) -- see SURVEY.md Appendix A.

The marlbase wrapper stack on top (TimeLimit -> RecordEpisodeStatistics -> CooperativeReward) is
restated in :class:`WrappedForaging` from marlbase/utils/wrappers.py:13-45,106-108 and
marlbase/utils/envs.py:93-109.
"""
from __future__ import annotations

from collections import defaultdict
from dataclasses import dataclass

import numpy as np

NONE, NORTH, SOUTH, WEST, EAST, LOAD = range(6)
_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_MASK = 0xFFFFFFFF
TAG_RESET = 0x52455345


def philox4x32_10(ctr, key):
    """Random123 Philox4x32-10; ``ctr`` 4 words, ``key`` 2 words -> 4 words."""
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for _ in range(10):
        p0 = _M0 * c0
        p1 = _M1 * c2
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & _MASK, (p0 >> 32) ^ c3 ^ k1, p0 & _MASK
        k0 = (k0 + _W0) & _MASK
        k1 = (k1 + _W1) & _MASK
    return c0, c1, c2, c3


class DrawStream:
    """Sequential 32-bit draws for one (seed, env, episode) reset; draw i = word i%4 of block i//4."""

    def __init__(self, seed, env_gid, episode_idx):
        self.key = (seed & _MASK, ((seed >> 32) & _MASK) ^ TAG_RESET)
        self.gid, self.ep, self.n = env_gid & _MASK, episode_idx & _MASK, 0

    def next_u32(self):
        block = philox4x32_10((self.gid, self.ep, self.n >> 2, 0), self.key)
        v = block[self.n & 3]
        self.n += 1
        return v

    def integers(self, lo, hi):
        return lo + ((self.next_u32() * (hi - lo)) >> 32)


@dataclass
class LBFConfig:
    rows: int = 8
    cols: int = 8
    n_agents: int = 2
    max_num_food: int = 3
    sight: int = 8
    min_player_level: int = 1
    max_player_level: int = 2
    min_food_level: int = 1
    max_food_level: int = 0  # <=0: None
    max_episode_steps: int = 50
    time_limit: int = 25
    force_coop: int = 0
    normalize_reward: int = 1
    cooperative_reward: int = 0
    penalty: float = 0.0
    observe_id: int = 0
    standardise_rewards: int = 0
    upstream_reset: int = 0   # 1: stale previous-episode positions block cells while spawning, the level-bound permutations consume draws

    @property
    def base_obs_dim(self):
        return 3 * self.max_num_food + 3 * self.n_agents

    @property
    def obs_dim(self):
        return self.base_obs_dim + (self.n_agents if self.observe_id else 0)


class _Player:
    def __init__(self):
        self.position = None
        self.level = None
        self.reward = 0.0


class ForagingRef:
    def __init__(self, cfg: LBFConfig):
        self.cfg = cfg
        self.players = [_Player() for _ in range(cfg.n_agents)]
        self.field = np.zeros((cfg.rows, cfg.cols), np.int32)
        self.current_step = 0
        self.food_spawned = 0

    # ---- spawning -------------------------------------------------------------------------
    def _is_empty(self, row, col, placed):
        if self.field[row, col] != 0:
            return False
        if self.cfg.upstream_reset:   # upstream _is_empty_location: every player that has a position, re-placed in this reset() or not
            placed = [p for p in self.players if p.position is not None]
        return all(p.position != (row, col) for p in placed)

    def reset(self, seed, env_gid, episode_idx):
        c = self.cfg
        rng = DrawStream(seed, env_gid, episode_idx)
        self.field[:] = 0
        placed = []
        if c.upstream_reset:
            for k in range(c.n_agents - 1, 0, -1):   # spawn_players: np_random.permutation over the (identical) level bounds
                rng.integers(0, k + 1)
        for p in self.players:
            p.reward = 0.0
            if not c.upstream_reset:
                p.position = None
            found = False
            for _ in range(1000):
                row, col = rng.integers(0, c.rows), rng.integers(0, c.cols)
                if self._is_empty(row, col, placed):
                    p.position, found = (row, col), True
                    p.level = rng.integers(c.min_player_level, c.max_player_level + 1)
                    break
            if not found:   # never reached for sane sizes; deterministic fallback shared by the three implementations: first empty cell, min level
                p.position, p.level = next((r, q) for r in range(c.rows) for q in range(c.cols) if self._is_empty(r, q, placed)), c.min_player_level
            placed.append(p)
        levels = sorted(p.level for p in self.players)
        max_lvl = c.max_food_level if c.max_food_level > 0 else sum(levels[:3])
        min_lvl = max_lvl if c.force_coop else c.min_food_level
        if c.upstream_reset:
            for k in range(c.max_num_food - 1, 0, -1):   # spawn_food: np_random.permutation over the food level bounds
                rng.integers(0, k + 1)
        count = attempts = 0
        while count < c.max_num_food and attempts < 1000:
            attempts += 1
            row, col = rng.integers(1, c.rows - 1), rng.integers(1, c.cols - 1)
            box = self.field[max(row - 1, 0) : row + 2, max(col - 1, 0) : col + 2].sum()
            cross = self.field[max(row - 2, 0) : row + 3, col].sum() + self.field[row, max(col - 2, 0) : col + 3].sum()
            if box > 0 or cross > 0 or not self._is_empty(row, col, self.players):
                continue
            self.field[row, col] = min_lvl if min_lvl == max_lvl else rng.integers(min_lvl, max_lvl + 1)
            count += 1
        self.food_spawned = int(self.field.sum())
        self.current_step = 0

    # ---- transition -----------------------------------------------------------------------
    def _adjacent_food(self, row, col):
        f, c = self.field, self.cfg
        return f[max(row - 1, 0), col] + f[min(row + 1, c.rows - 1), col] + f[row, max(col - 1, 0)] + f[row, min(col + 1, c.cols - 1)]

    def _adjacent_food_location(self, row, col):
        f, c = self.field, self.cfg
        if row > 1 and f[row - 1, col] > 0:
            return row - 1, col
        if row < c.rows - 1 and f[row + 1, col] > 0:
            return row + 1, col
        if col > 1 and f[row, col - 1] > 0:
            return row, col - 1
        if col < c.cols - 1 and f[row, col + 1] > 0:
            return row, col + 1
        return None

    def _valid(self, p, a):
        (row, col), f, c = p.position, self.field, self.cfg
        if a == NONE:
            return True
        if a == NORTH:
            return row > 0 and f[row - 1, col] == 0
        if a == SOUTH:
            return row < c.rows - 1 and f[row + 1, col] == 0
        if a == WEST:
            return col > 0 and f[row, col - 1] == 0
        if a == EAST:
            return col < c.cols - 1 and f[row, col + 1] == 0
        if a == LOAD:
            return self._adjacent_food(row, col) > 0
        return False

    def step(self, actions, load_order=None):
        """`load_order`: optional permutation of the loading players' indices (upstream pops an unordered Python set, SURVEY H2);
        default = ascending agent index, the order the C oracle and the CUDA kernel fix."""
        c = self.cfg
        self.current_step += 1
        for p in self.players:
            p.reward = 0.0
        actions = [a if self._valid(p, a) else NONE for p, a in zip(self.players, actions)]
        delta = {NONE: (0, 0), NORTH: (-1, 0), SOUTH: (1, 0), WEST: (0, -1), EAST: (0, 1), LOAD: (0, 0)}
        collisions = defaultdict(list)
        loading = []
        for idx, (p, a) in enumerate(zip(self.players, actions)):
            dr, dc = delta[a]
            collisions[(p.position[0] + dr, p.position[1] + dc)].append(p)
            if a == LOAD:
                loading.append(idx)
        for cell, who in collisions.items():
            if len(who) == 1:
                who[0].position = cell
        pending = set(loading)
        if load_order is not None:
            assert sorted(load_order) == loading, "load_order must be a permutation of the loading players"
            loading = list(load_order)
        for idx in loading:  # ascending agent index; upstream pops an unordered set
            if idx not in pending:
                continue
            player = self.players[idx]
            loc = self._adjacent_food_location(*player.position)
            pending.discard(idx)
            if loc is None:
                continue
            frow, fcol = loc
            food = int(self.field[frow, fcol])
            adj = [
                j
                for j, q in enumerate(self.players)
                if (abs(q.position[0] - frow) == 1 and q.position[1] == fcol or abs(q.position[1] - fcol) == 1 and q.position[0] == frow)
                and (j in pending or j == idx)
            ]
            level_sum = sum(self.players[j].level for j in adj)
            pending -= set(adj)
            if level_sum < food:
                for j in adj:
                    self.players[j].reward -= c.penalty
                continue
            for j in adj:
                r = float(self.players[j].level * food)
                if c.normalize_reward:
                    r = r / float(level_sum * self.food_spawned)
                self.players[j].reward = r
            self.field[frow, fcol] = 0
        done = bool(self.field.sum() == 0 or c.max_episode_steps <= self.current_step)
        return [p.reward for p in self.players], done

    # ---- observation ----------------------------------------------------------------------
    def obs(self, agent):
        c = self.cfg
        me = self.players[agent]
        s = c.sight
        r0, c0 = max(me.position[0] - s, 0), max(me.position[1] - s, 0)
        window = self.field[r0 : min(me.position[0] + s + 1, c.rows), c0 : min(me.position[1] + s + 1, c.cols)]
        out = np.zeros(c.base_obs_dim, np.float32)
        out[: 3 * c.max_num_food] = np.tile(np.array([-1, -1, 0], np.float32), c.max_num_food)
        out[3 * c.max_num_food :] = np.tile(np.array([-1, -1, 0], np.float32), c.n_agents)
        for i, (y, x) in enumerate(zip(*np.nonzero(window))):
            out[3 * i : 3 * i + 3] = (y, x, window[y, x])

        def transform(pos):
            return (pos[0] - me.position[0] + min(s, me.position[0]), pos[1] - me.position[1] + min(s, me.position[1]))

        seen = [(transform(q.position), q.level, q is me) for q in self.players]
        seen = [t for t in seen if min(t[0]) >= 0 and max(t[0]) <= 2 * s]
        seen = [t for t in seen if t[2]] + [t for t in seen if not t[2]]
        for i, (pos, lvl, _) in enumerate(seen):
            out[3 * c.max_num_food + 3 * i : 3 * c.max_num_food + 3 * i + 3] = (pos[0], pos[1], lvl)
        return out

    # ---- (de)serialisation into the int8 layout the C oracle and the kernel use -------------
    def export(self):
        c = self.cfg
        players = np.zeros((c.n_agents, 4), np.int8)
        for i, p in enumerate(self.players):
            players[i, :3] = (p.position[0], p.position[1], p.level)
        return self.field.astype(np.int8).reshape(-1).copy(), players

    def load(self, field, players, step, food_spawned):
        c = self.cfg
        self.field = np.asarray(field, np.int32).reshape(c.rows, c.cols).copy()
        for i, p in enumerate(self.players):
            p.position, p.level = (int(players[i][0]), int(players[i][1])), int(players[i][2])
        self.current_step, self.food_spawned = int(step), int(food_spawned)


class StandardiseReward:
    """marlbase's StandardiseReward wrapper (wrappers.py:111-141): per-agent running reward statistics."""

    def __init__(self, n_agents):
        # StandardiseReward.__init__ (wrappers.py:112-117)
        self.stdr_wrp_sumw = np.zeros(n_agents, dtype=np.float32)
        self.stdr_wrp_wmean = np.zeros(n_agents, dtype=np.float32)
        self.stdr_wrp_t = np.zeros(n_agents, dtype=np.float32)
        self.stdr_wrp_n = 0

    def reward(self, reward):
        """StandardiseReward.reward (wrappers.py:119-141), verbatim arithmetic"""
        weight = 1.0
        q = reward - self.stdr_wrp_wmean
        temp_sumw = self.stdr_wrp_sumw + weight
        r = q * weight / temp_sumw
        self.stdr_wrp_wmean += r
        self.stdr_wrp_t += q * r * self.stdr_wrp_sumw
        self.stdr_wrp_sumw = temp_sumw
        self.stdr_wrp_n += 1
        if self.stdr_wrp_n == 1:
            return reward
        var = (self.stdr_wrp_t * self.stdr_wrp_n) / (self.stdr_wrp_sumw * (self.stdr_wrp_n - 1))
        return (reward - self.stdr_wrp_wmean) / (np.sqrt(var) + 1e-6)


class WrappedForaging:
    """ForagingRef under marlbase's wrapper stack: TimeLimit(time_limit) -> RecordEpisodeStatistics -> [ObserveID] -> [StandardiseReward] ->
    [CooperativeReward]  (marlbase/utils/envs.py:93-109).  The two optional wrappers transcribe the reference's numpy code literally
    (wrappers.py:96-103 and 119-141): they are what pins the C restatement and the kernel for these two flags."""

    def __init__(self, cfg: LBFConfig, seed: int, env_gid: int = 0):
        self.cfg, self.seed, self.gid = cfg, seed, env_gid
        self.env = ForagingRef(cfg)
        self.n_resets = 0
        self.episode_reward = np.zeros(cfg.n_agents, np.float32)
        self.episode_length = 0
        self.stdr = StandardiseReward(cfg.n_agents)

    def _observation(self):
        observation = tuple(self.env.obs(i) for i in range(self.cfg.n_agents))
        if self.cfg.observe_id:   # ObserveID.observation (wrappers.py:96-103)
            n_agents = self.cfg.n_agents
            observation = np.stack(observation)
            observation = np.concatenate((np.eye(n_agents, dtype=observation.dtype), observation), axis=1)
            observation = tuple(o.squeeze() for o in np.split(observation, n_agents))
        return observation

    def reset(self):
        self.env.reset(self.seed, self.gid, self.n_resets)
        self.n_resets += 1
        self.episode_reward = np.zeros(self.cfg.n_agents, np.float32)
        self.episode_length = 0
        return self._observation(), {}

    def step(self, actions):
        c = self.cfg
        reward, done = self.env.step(list(actions))
        truncated = bool(c.time_limit > 0 and self.env.current_step >= c.time_limit)  # gymnasium TimeLimit
        info = {}
        self.episode_reward = self.episode_reward + np.array(reward, dtype=np.float32)  # wrappers.py:33
        self.episode_length += 1
        if done or truncated:
            info["episode_returns"] = self.episode_reward.copy()
            for i, r in enumerate(self.episode_reward):
                info[f"agent{i}/episode_returns"] = r
            info["episode_length"] = self.episode_length
        if c.standardise_rewards:
            reward = self.stdr.reward(reward)
        if c.cooperative_reward:
            reward = c.n_agents * [sum(reward)]  # wrappers.py:106-108
        return self._observation(), reward, done, truncated, info

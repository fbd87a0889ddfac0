"""CPU restatement of the multi-robot warehouse (third-party ``rware`` 2.x ``Warehouse``) under marlbase's wrapper stack -- pure
Python / numpy, one env per object.  TEST INFRASTRUCTURE ONLY: the CUDA kernel (codebase_b200/csrc/rware_env.cu) is checked against it
bit for bit.  PARITY UNPINNED against upstream ``rware`` (third-party, absent from the reference checkout): the semantics are the ones
DESIGN.md Appendix B restates from memory.

Move resolution is written twice: ``resolve_moves`` is the closed-form rule the kernel implements (cycles, chains, merges) and
``resolve_moves_networkx`` transcribes upstream's ``networkx`` graph literally; a CPU test checks that the two agree.

Coordinates are (x = column, y = row); a cell's index is y * cols + x.  An agent is [x, y, dir, carried shelf id (0: none)].
"""
from __future__ import annotations

import numpy as np

from .lbf_ref import DrawStream, StandardiseReward, philox4x32_10

NOOP, FORWARD, LEFT, RIGHT, TOGGLE_LOAD = range(5)
UP, DOWN, DIR_LEFT, DIR_RIGHT = range(4)
TURN_CYCLE = (UP, DIR_RIGHT, DOWN, DIR_LEFT)   # RIGHT turns one step forward in this cycle, LEFT one step back
TAG_REQUEST = 0x52455155                      # replacement requests: key (seed_lo, seed_hi ^ tag), ctr (env_gid, episode, step, goal)
EMPTY_CELL_DIRECTION = (1.0, 0.0, 0.0, 0.0)   # (recalled quirk) the direction one-hot written for a sensor cell without an agent
_MASK = 0xFFFFFFFF


def is_highway(cfg, x, y):
    rows, cols = cfg.rows, cfg.cols
    return (x % 3 == 0 or y % (cfg.column_height + 1) == 0 or y == rows - 1
            or (y > rows - (cfg.column_height + 3) and x in (cols // 2 - 1, cols // 2)))


def home_shelves(cfg):
    """uint8 [rows*cols]: shelf ids 1.. in row-major order on every non-highway cell."""
    g = np.zeros(cfg.rows * cfg.cols, np.uint8)
    k = 0
    for y in range(cfg.rows):
        for x in range(cfg.cols):
            if not is_highway(cfg, x, y):
                k += 1
                g[y * cfg.cols + x] = k
    return g


def n_shelves(cfg):
    return int((home_shelves(cfg) > 0).sum())


def goals(cfg):
    return [(cfg.cols // 2 - 1, cfg.rows - 1), (cfg.cols // 2, cfg.rows - 1)]


def forward_cell(cfg, x, y, d):
    """FORWARD's target, clamped at the border."""
    if d == UP:
        return x, max(0, y - 1)
    if d == DOWN:
        return x, min(cfg.rows - 1, y + 1)
    if d == DIR_LEFT:
        return max(0, x - 1), y
    return min(cfg.cols - 1, x + 1), y


def turn(d, step):
    return TURN_CYCLE[(TURN_CYCLE.index(d) + step) % 4]


def resolve_moves(cfg, agents, shelves, actions, tie_rank=None):
    """Closed form of upstream's move resolution.  Returns the actions after cancellation (uncommitted FORWARD -> NOOP).

    Every agent has one edge, from its cell to its target (a self-loop unless it moves), so each weakly connected component holds at most
    one cycle.  A cycle of length 2 commits nobody, any other cycle commits exactly its agents, and a component without a cycle is an
    in-tree towards one empty cell whose committed agents are those on networkx's dag_longest_path: walking back from the empty cell it
    takes, at each node, the predecessor with the longest chain behind it.  On a tie this rule takes the agent whose cell entered the graph
    first (the graph is built in agent order, start cell then target cell); `tie_rank` (one integer per agent, lowest wins) replaces that
    order.  networkx itself breaks the tie by the iteration order of the component's node set (see DESIGN.md Appendix B)."""
    N, C = len(agents), cfg.cols
    act = [int(a) for a in actions]
    cell = [y * C + x for x, y, _, _ in agents]
    occ = {c: i for i, c in enumerate(cell)}
    tgt = []
    for i, (x, y, d, s) in enumerate(agents):
        t = cell[i]
        if act[i] == FORWARD:
            tx, ty = forward_cell(cfg, x, y, d)
            t = ty * C + tx
            if s and t != cell[i] and shelves[t] and not (t in occ and agents[occ[t]][3]):
                act[i], t = NOOP, cell[i]   # a loaded agent cannot enter a cell holding a resting shelf
        tgt.append(t)
    nxt = [occ.get(t, -1) for t in tgt]
    rank = [2 * u for u in range(N)]   # insertion position of the agent's cell as a graph node
    for u in range(N):
        first = next((i for i in range(u) if tgt[i] == cell[u]), None)
        if first is not None:
            rank[u] = 2 * first + 1
    if tie_rank is not None:
        rank = list(tie_rank)
    depth, cyc_len, chain = [0] * N, [0] * N, []
    for v in range(N):
        x, path = v, [v]
        for k in range(1, N + 1):
            x = nxt[x]
            if x < 0:
                break
            depth[x] = max(depth[x], k)
            if x == v and not cyc_len[v]:
                cyc_len[v] = k
            path.append(x)
        chain.append(path if x < 0 else None)   # None: the chain runs into a cycle
    key = [(depth[u], -rank[u]) for u in range(N)]
    win = [all(key[u] >= key[j] for j in range(N) if tgt[j] == tgt[u]) for u in range(N)]
    for v in range(N):
        if cyc_len[v]:
            ok = cyc_len[v] != 2
        elif chain[v] is not None:
            ok = all(win[x] for x in chain[v])
        else:
            ok = False
        if not ok and act[v] == FORWARD:
            act[v] = NOOP
    return act


def resolve_moves_networkx(cfg, agents, shelves, actions):
    """Upstream's resolution transcribed literally (rware Warehouse.step with a networkx.DiGraph on (x, y) cells).  Returns the actions and,
    per agent, the position of its cell in its component's node order (the order dag_longest_path breaks ties in)."""
    import networkx as nx

    act = [int(a) for a in actions]
    grid_agents = {(x, y): i + 1 for i, (x, y, _, _) in enumerate(agents)}
    G = nx.DiGraph()
    for i, (x, y, d, s) in enumerate(agents):
        start = (x, y)
        target = forward_cell(cfg, x, y, d) if act[i] == FORWARD else start
        if (s and start != target and shelves[target[1] * cfg.cols + target[0]]
                and not (target in grid_agents and agents[grid_agents[target] - 1][3])):
            act[i] = NOOP
            G.add_edge(start, start)
        else:
            G.add_edge(start, target)
    commited = set()
    node_pos = {}
    for comp in [G.subgraph(c).copy() for c in nx.weakly_connected_components(G)]:
        node_pos.update({n: k for k, n in enumerate(comp.nodes)})
        try:
            cycle = nx.algorithms.find_cycle(comp)
            if len(cycle) == 2:
                continue
            for edge in cycle:
                commited.add(edge[0])
        except nx.NetworkXNoCycle:
            for node in nx.algorithms.dag_longest_path(comp):
                commited.add(node)
    commited_agents = {grid_agents[c] - 1 for c in commited if c in grid_agents}
    for i in set(range(len(agents))) - commited_agents:
        assert act[i] == FORWARD
        act[i] = NOOP
    return act, [node_pos[(x, y)] for x, y, _, _ in agents]


class Warehouse:
    """One warehouse: agents [N][4], shelves uint8 [rows*cols] (shelf id at its current cell, a carried shelf at its carrier's),
    requested bool [n_shelves + 1], step, inactive (steps since the last delivery)."""

    def __init__(self, cfg):
        self.cfg = cfg
        self.home = home_shelves(cfg)
        self.n_shelves = int((self.home > 0).sum())
        self.highway = np.array([is_highway(cfg, x, y) for y in range(cfg.rows) for x in range(cfg.cols)])
        self.agents = [[0, 0, UP, 0] for _ in range(cfg.n_agents)]
        self.shelves = self.home.copy()
        self.requested = np.zeros(self.n_shelves + 1, bool)
        self.step_count = self.inactive = 0

    def reset(self, seed, env_gid, episode_idx):
        c = self.cfg
        ds = DrawStream(seed, env_gid, episode_idx)
        taken = set()
        for a in self.agents:
            while True:
                p = ds.integers(0, c.rows * c.cols)
                if p not in taken:
                    break
            taken.add(p)
            a[0], a[1], a[3] = p % c.cols, p // c.cols, 0
        for a in self.agents:
            a[2] = ds.integers(0, 4)
        self.requested[:] = False
        for _ in range(c.request_queue_size):
            while True:
                s = 1 + ds.integers(0, self.n_shelves)
                if not self.requested[s]:
                    break
            self.requested[s] = True
        self.shelves = self.home.copy()
        self.step_count = self.inactive = 0

    def step(self, actions, seed, env_gid, episode):
        """Returns (rewards [N] floats, terminated)."""
        c, C = self.cfg, self.cfg.cols
        act = resolve_moves(c, self.agents, self.shelves, [a if 0 <= a < 5 else NOOP for a in actions])
        moving = [i for i in range(len(self.agents)) if act[i] == FORWARD]
        carried = [(self.agents[i][3], *forward_cell(c, *self.agents[i][:3])) for i in moving if self.agents[i][3]]
        for i in moving:
            if self.agents[i][3]:
                self.shelves[self.agents[i][1] * C + self.agents[i][0]] = 0
        for s, x, y in carried:
            self.shelves[y * C + x] = s
        for i, a in enumerate(self.agents):
            if act[i] == FORWARD:
                a[0], a[1] = forward_cell(c, a[0], a[1], a[2])
            elif act[i] == LEFT:
                a[2] = turn(a[2], -1)
            elif act[i] == RIGHT:
                a[2] = turn(a[2], +1)
            elif act[i] == TOGGLE_LOAD:
                here = a[1] * C + a[0]
                if not a[3]:
                    a[3] = int(self.shelves[here])
                elif not self.highway[here]:
                    a[3] = 0
        self.step_count += 1
        rewards = [0.0] * len(self.agents)
        delivered = False
        for g, (gx, gy) in enumerate(goals(c)):
            s = int(self.shelves[gy * C + gx])
            if not s or not self.requested[s]:
                continue
            delivered = True
            free = np.nonzero(~self.requested[1:])[0] + 1   # shelves not requested before the replacement
            key = (seed & _MASK, ((seed >> 32) & _MASK) ^ TAG_REQUEST)
            u = philox4x32_10((env_gid & _MASK, episode & _MASK, self.step_count, g), key)[0]
            new = int(free[(u * len(free)) >> 32])
            self.requested[s], self.requested[new] = False, True
            who = next(i for i, a in enumerate(self.agents) if (a[0], a[1]) == (gx, gy))
            rewards[who] += 1.0
        self.inactive = 0 if delivered else self.inactive + 1
        done = bool((c.max_inactivity_steps and self.inactive >= c.max_inactivity_steps) or (c.max_steps and self.step_count >= c.max_steps))
        return rewards, done

    def obs(self, agent):
        c = self.cfg
        x, y, d, s = self.agents[agent]
        out = [float(x), float(y), float(s != 0), *[float(d == k) for k in range(4)], float(self.highway[y * c.cols + x])]
        where = {(a[0], a[1]): a for a in self.agents}
        r = c.sensor_range
        for yy in range(y - r, y + r + 1):
            for xx in range(x - r, x + r + 1):
                inside = 0 <= xx < c.cols and 0 <= yy < c.rows
                other = where.get((xx, yy)) if inside else None
                out += [0.0, *EMPTY_CELL_DIRECTION] if other is None else [1.0, *[float(other[2] == k) for k in range(4)]]
                sid = int(self.shelves[yy * c.cols + xx]) if inside else 0
                out += [1.0, float(self.requested[sid])] if sid else [0.0, 0.0]
        return np.array(out, np.float32)

    # ---- the kernel's state layout -------------------------------------------------------------
    def export(self):
        req = np.zeros(8, np.uint32)
        for k in np.nonzero(self.requested)[0]:
            req[k >> 5] |= np.uint32(1 << (k & 31))
        return self.shelves.copy(), np.array(self.agents, np.uint8).reshape(-1, 4), req.view(np.int32)

    def load(self, shelves, agents, requested, step, inactive):
        self.shelves = np.asarray(shelves, np.uint8).reshape(-1).copy()
        self.agents = [[int(v) for v in a] for a in np.asarray(agents).reshape(-1, 4)]
        bits = np.asarray(requested).astype(np.uint32)
        self.requested = np.array([bool((int(bits[k >> 5]) >> (k & 31)) & 1) for k in range(self.n_shelves + 1)])
        self.step_count, self.inactive = int(step), int(inactive)


class WrappedWarehouse:
    """Warehouse under marlbase's wrapper stack: TimeLimit(time_limit) -> RecordEpisodeStatistics -> [ObserveID] -> [StandardiseReward] ->
    [CooperativeReward] (marlbase/utils/envs.py:93-109), the optional wrappers' arithmetic as oracle/lbf_ref.WrappedForaging has it."""

    def __init__(self, cfg, seed, env_gid=0):
        self.cfg, self.seed, self.gid = cfg, seed, env_gid
        self.env = Warehouse(cfg)
        self.n_resets = 0
        self.episode_reward = np.zeros(cfg.n_agents, np.float32)
        self.episode_length = 0
        self.stdr = StandardiseReward(cfg.n_agents)

    def observation(self):
        obs = np.stack([self.env.obs(i) for i in range(self.cfg.n_agents)])
        if self.cfg.observe_id:
            obs = np.concatenate((np.eye(self.cfg.n_agents, dtype=obs.dtype), obs), axis=1)
        return obs

    def reset(self):
        self.env.reset(self.seed, self.gid, self.n_resets)
        self.n_resets += 1
        self.episode_reward = np.zeros(self.cfg.n_agents, np.float32)
        self.episode_length = 0
        return self.observation()

    def step(self, actions):
        """Returns (obs [N][D], rewards float32 [N], terminated, truncated, info)."""
        c = self.cfg
        reward, done = self.env.step(list(actions), self.seed, self.gid, self.n_resets - 1)
        truncated = bool(c.time_limit > 0 and self.env.step_count >= c.time_limit)
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
        return self.observation(), np.asarray(reward, np.float32), done, truncated, info


class OracleVecRware:
    """E wrapped warehouses with the native handle's step semantics (autoreset in the same step, inactive envs after an ended episode)."""

    def __init__(self, cfg, E, seed, gid0=0):
        self.cfg, self.E, self.N, self.D = cfg, E, cfg.n_agents, cfg.obs_dim
        self.envs = [WrappedWarehouse(cfg, seed, gid0 + e) for e in range(E)]
        self.active = np.ones(E, np.uint8)

    @property
    def episode_idx(self):
        return np.array([w.n_resets for w in self.envs], np.int64)

    @property
    def step_count(self):
        return np.array([w.env.step_count for w in self.envs], np.int64)

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
            o, r, d, t, info = w.step(actions[e])
            rew[e], done[e], trunc[e] = r, d, t
            if d or t:
                fret[e], flen[e] = info["episode_returns"], info["episode_length"]
                if autoreset:
                    o = w.reset()
                else:
                    self.active[e] = 0
            obs[e] = o
        return obs, rew, done, trunc, fret, flen

    def state(self):
        sh, ag, rq = zip(*[w.env.export() for w in self.envs])
        return dict(shelves=np.stack(sh), agents=np.stack(ag), requested=np.stack(rq), step=self.step_count.astype(np.int32),
                    inactive=np.array([w.env.inactive for w in self.envs], np.int32),
                    ep_return=np.stack([w.episode_reward for w in self.envs]).astype(np.float32),
                    ep_len=np.array([w.episode_length for w in self.envs], np.int32), episode_idx=self.episode_idx.astype(np.int32),
                    active=self.active.copy())

"""Level-Based Foraging grid observations (``Foraging-grid-*`` ids) for the tests: the literal transcription of upstream's construction, the
C restatement (tests/lbf_grid_oracle.c) through ctypes, and a vectorised env oracle that puts them on top of oracle/lbf_c.py.

PARITY UNPINNED: ``lbforaging`` is not vendored.  ``grid_obs_upstream`` transcribes ``ForagingEnv._make_gym_obs`` with
``grid_observation=True`` as recalled (DESIGN.md Appendix A); tests/test_lbf_grid.py checks it against the installed package where one
can be imported.  Every recalled constant is in ``RECALLED``.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))

# Recalled from upstream lbforaging (DESIGN.md Appendix A)
RECALLED = dict(
    layers=("agents", "foods", "access"),   # np.stack order of make_global_grid_arrays
    dtype=np.float32,                        # every layer is float32; FlattenObservation keeps C order (layer, row, col)
    pad_value={"agents": 0.0, "foods": 0.0, "access": 0.0},
    grid_sights=lambda s: range(1, s + 1),   # grid ids are registered for every sight 1..s (the `-{k}s` tag is omitted at k = s)
)


def grid_obs_upstream(field, players, sight):
    """ForagingEnv._make_gym_obs, grid branch, transcribed: the global padded layers, then one window slice per agent.
    `field`: int [rows, cols]; `players`: [(row, col, level)] per agent.  Returns a tuple of float32 [3, 2k+1, 2k+1]."""
    field = np.asarray(field)
    grid_shape_x, grid_shape_y = field.shape
    grid_shape_x += 2 * sight
    grid_shape_y += 2 * sight
    grid_shape = (grid_shape_x, grid_shape_y)

    agents_layer = np.zeros(grid_shape, dtype=np.float32)
    for player_x, player_y, level in players:
        agents_layer[player_x + sight, player_y + sight] = level

    foods_layer = np.zeros(grid_shape, dtype=np.float32)
    foods_layer[sight:-sight, sight:-sight] = field.copy()

    access_layer = np.ones(grid_shape, dtype=np.float32)
    # out of bounds not accessible
    access_layer[:sight, :] = 0.0
    access_layer[-sight:, :] = 0.0
    access_layer[:, :sight] = 0.0
    access_layer[:, -sight:] = 0.0
    # agent locations are not accessible
    for player_x, player_y, _ in players:
        access_layer[player_x + sight, player_y + sight] = 0.0
    # food locations are not accessible
    foods_x, foods_y = field.nonzero()
    for x, y in zip(foods_x, foods_y):
        access_layer[x + sight, y + sight] = 0.0

    layers = np.stack([agents_layer, foods_layer, access_layer])

    def get_agent_grid_bounds(agent_x, agent_y):
        return agent_x, agent_x + 2 * sight + 1, agent_y, agent_y + 2 * sight + 1

    agents_bounds = [get_agent_grid_bounds(x, y) for x, y, _ in players]
    return tuple(layers[:, start_x:end_x, start_y:end_y] for start_x, end_x, start_y, end_y in agents_bounds)


def flat_upstream(field, players_i8, sight):
    """FlattenObservation of grid_obs_upstream: [N, D] float32 from the int8 layouts the kernels use (players [N][4])."""
    pl = [(int(p[0]), int(p[1]), int(p[2])) for p in players_i8]
    return np.stack([o.reshape(-1) for o in grid_obs_upstream(field, pl, sight)]).astype(np.float32)


# ---- the C restatement ------------------------------------------------------------------------------------------------------------------------
_LIB = None


def lib():
    """tests/lbf_grid_oracle.c compiled once per process into a temporary directory (nothing is written into the tree)."""
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="lbf_grid_oracle_"), "liblbf_grid_oracle.so")
        subprocess.check_call([os.environ.get("CC", "gcc"), "-O2", "-fPIC", "-Wall", "-Wextra", "-Werror", "-std=c11", "-shared", "-o", out,
                               os.path.join(_HERE, "lbf_grid_oracle.c")])
        _LIB = C.CDLL(out)
    return _LIB


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def grid_obs_c(rows, cols, sight, field, players):
    """field int8 [E][rows*cols], players int8 [E][N][4] -> float32 [E][N][D]."""
    field = np.ascontiguousarray(field, np.int8).reshape(-1, rows * cols)
    players = np.ascontiguousarray(players, np.int8)
    E, N = players.shape[0], players.shape[1]
    D = lib().lbf_grid_obs_dim(C.c_int(sight))
    out = np.zeros((E, N, D), np.float32)
    lib().lbf_grid_obs_batch(C.c_int(E), C.c_int(rows), C.c_int(cols), C.c_int(N), C.c_int(sight), _p(field), _p(players), _p(out))
    return out


class GridOracleVecEnv:
    """oracle/lbf_c.OracleVecEnv with the grid observation: the transition (and autoreset) of the C oracle, whose observations are replaced by
    grid_obs_c of the state it leaves -- the grid observation is built from the same post-step / post-reset state as the vector one."""

    def __init__(self, cfgkw: dict, n_envs: int, seed: int, env_gid0: int = 0):
        from oracle import lbf_c

        kw = {k: v for k, v in cfgkw.items() if k != "grid_observation"}
        self.env = lbf_c.OracleVecEnv(lbf_c.make_cfg(**kw), n_envs, seed, env_gid0)
        c = self.env.cfg
        self.rows, self.cols, self.sight, self.N = c.rows, c.cols, c.sight, c.n_agents
        self.D = 3 * (2 * self.sight + 1) ** 2

    def __getattr__(self, name):
        return getattr(self.__dict__["env"], name)

    def obs(self):
        return grid_obs_c(self.rows, self.cols, self.sight, self.env.field, self.env.players)

    def reset(self, mask=None):
        self.env.reset(mask)
        return self.obs()

    def step(self, actions, autoreset=False):
        _, rew, done, trunc, fret, flen = self.env.step(actions, autoreset)
        return self.obs(), rew, done, trunc, fret, flen

    def set_state(self, *args, **kwargs):
        self.env.set_state(*args, **kwargs)

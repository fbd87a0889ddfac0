"""Low-level Python handle over the native LBF env (marl_lbf_* entry points of libmarlb200.so).

All arrays are torch CUDA tensors; nothing here computes on the CPU.  Env ids follow the third-party
``lbforaging`` registration the reference passes to ``gym.make`` (marlbase/utils/envs.py:90-92,
README.md:80-85): ``[lbforaging:]Foraging[-grid][-{k}s]-{s}x{s}-{p}p-{f}f[-coop][-pen]-v{1,2,3}``.  Vector-observation ids take
``-2s`` only; grid-observation ids (``-grid``) any sight 1 <= k <= s, and sight s without the tag (DESIGN.md Appendix A).
"""
from __future__ import annotations

import math
import re
from dataclasses import dataclass, asdict

import torch

from . import _native as nat
from .native_env import NativeEnv, TrajStore  # noqa: F401  (callers import TrajStore from here too)

_ID = re.compile(r"^(?:lbforaging:)?Foraging(?P<grid>-grid)?(?:-(?P<k>\d+)s)?-(?P<s>\d+)x(?P<s2>\d+)-(?P<p>\d+)p-(?P<f>\d+)f(?P<coop>-coop)?(?P<pen>-pen)?-v(?P<v>\d+)$")


@dataclass
class LbfConfig:
    rows: int = 8
    cols: int = 8
    n_agents: int = 2
    max_num_food: int = 3
    sight: int = 8
    min_player_level: int = 1
    max_player_level: int = 2
    min_food_level: int = 1
    max_food_level: int = 0
    max_episode_steps: int = 50
    time_limit: int = 25
    force_coop: int = 0
    normalize_reward: int = 1
    cooperative_reward: int = 0
    penalty: float = 0.0
    observe_id: int = 0            # env.observe_id: ObserveID wrapper (one-hot agent id in front of every observation)
    standardise_rewards: int = 0   # env.standardise_rewards: StandardiseReward wrapper (per-env running statistics)
    upstream_reset: int = 0        # 1: upstream's reset details (stale positions block cells, permutation draws consumed), see marl_lbf_cfg
    grid_observation: int = 0      # 1: grid observation (Foraging-grid-* ids): agents | foods | access layers of the window, flattened

    @property
    def obs_dim(self) -> int:
        if self.grid_observation:
            return 3 * (2 * self.sight + 1) ** 2
        return 3 * self.max_num_food + 3 * self.n_agents + (self.n_agents if self.observe_id else 0)

    @property
    def n_actions(self) -> int:
        return 6

    @property
    def obs_bounds(self) -> tuple[float, float]:
        """Observation-space bounds: coordinates and levels, -1 for absent entities.  A grid observation is only served flattened, and
        FlattenObservation's Box is unbounded."""
        if self.grid_observation:
            return -math.inf, math.inf
        return -1.0, float(max(self.rows, self.cols))

    def to_native(self) -> nat.LbfCfg:
        return nat.LbfCfg(**asdict(self))


def parse_env_id(name: str, time_limit: int = 0, **overrides) -> LbfConfig:
    m = _ID.match(name)
    if not m:
        raise ValueError(f"unsupported environment id {name!r}: the GPU path implements Level-Based Foraging ids only")
    s, s2, p, f, v = int(m["s"]), int(m["s2"]), int(m["p"]), int(m["f"]), int(m["v"])
    grid, k = bool(m["grid"]), (int(m["k"]) if m["k"] is not None else None)
    if k is not None and not grid and k != 2:
        raise ValueError(f"unsupported environment id {name!r}: the GPU path implements Level-Based Foraging ids only")
    if grid and k is not None and not 1 <= k <= s:
        raise ValueError(f"environment id {name!r}: grid ids take a sight 1 <= k <= {s} (the field size), got -{k}s")
    cfg = LbfConfig(rows=s, cols=s2, n_agents=p, max_num_food=f, sight=k if k is not None else s,
                    max_player_level=2 if v >= 3 else 3, force_coop=int(bool(m["coop"])),
                    penalty=0.1 if m["pen"] else 0.0, time_limit=int(time_limit or 0), grid_observation=int(grid))
    for k, val in overrides.items():
        if not hasattr(cfg, k):
            raise TypeError(f"unknown LBF option {k!r}")
        setattr(cfg, k, val)
    return cfg


class NativeLbf(NativeEnv):
    PREFIX = "lbf"

    def _env_fields(self):
        return (("field", torch.int8, (self.cfg.rows * self.cfg.cols,)), ("players", torch.int8, (self.N, 4)), ("step", torch.int32, ()),
                ("food_spawned", torch.int32, ()))

    def set_state(self, field: torch.Tensor, players: torch.Tensor, step: torch.Tensor):
        self._set_state(field, players, step)

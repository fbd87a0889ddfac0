"""Low-level Python handle over the native multi-robot warehouse env (marl_rware_* entry points of libmarlb200.so).

All arrays are torch CUDA tensors; nothing here computes on the CPU.  Env ids follow the third-party ``rware`` 2.x registration
(gymnasium) the reference's README recommends: ``[rware:]rware-{size}-{N}ag[-easy|-hard]-v2``.  The constructor arguments of those ids
are recalled, not checked against the package (DESIGN.md Appendix B); every recalled value is a named constant below or a config field,
so a correction is a one-line change.
"""
from __future__ import annotations

import re
from dataclasses import dataclass, asdict

import torch

from . import _native as nat
from .native_env import NativeEnv

_ID = re.compile(r"^(?:rware:)?rware-(?P<size>[a-z]+)-(?P<n>\d+)ag(?:-(?P<diff>easy|hard))?-v(?P<v>\d+)$")

SIZES = {"tiny": (1, 3), "small": (2, 3), "medium": (2, 5), "large": (3, 5)}   # (shelf_rows, shelf_columns)
DIFFICULTY = {"easy": 2.0, None: 1.0, "hard": 0.5}                               # request_queue_size = int(N x this)
COLUMN_HEIGHT = 8            # (recalled)
SENSOR_RANGE = 1             # (recalled)
MAX_STEPS = 500              # (recalled)
MAX_INACTIVITY_STEPS = None  # (recalled) None: no inactivity limit
MAX_AGENTS = 19
_OVERRIDES = ("column_height", "shelf_rows", "shelf_columns", "request_queue_size", "max_steps", "max_inactivity_steps", "sensor_range")


@dataclass
class RwareConfig:
    shelf_rows: int = 1
    shelf_columns: int = 3
    column_height: int = COLUMN_HEIGHT
    n_agents: int = 4
    request_queue_size: int = 4
    max_steps: int = MAX_STEPS
    max_inactivity_steps: int = 0  # 0: None
    sensor_range: int = SENSOR_RANGE
    time_limit: int = 0            # TimeLimit wrapper, env.time_limit; 0 = absent
    cooperative_reward: int = 0    # CooperativeReward wrapper
    observe_id: int = 0            # ObserveID wrapper
    standardise_rewards: int = 0   # StandardiseReward wrapper

    @property
    def rows(self) -> int:
        return (self.column_height + 1) * self.shelf_rows + 2

    @property
    def cols(self) -> int:
        return 3 * self.shelf_columns + 1

    @property
    def obs_dim(self) -> int:
        return 8 + 7 * (2 * self.sensor_range + 1) ** 2 + (self.n_agents if self.observe_id else 0)

    @property
    def n_actions(self) -> int:
        return 5

    @property
    def obs_bounds(self) -> tuple[float, float]:
        """Observation-space bounds: coordinates, the rest 0 / 1."""
        return 0.0, float(max(self.rows, self.cols) - 1)

    def to_native(self) -> nat.RwareCfg:
        return nat.RwareCfg(**asdict(self))


def is_rware_id(name: str) -> bool:
    return str(name).split(":")[-1].startswith("rware-")


def parse_rware_id(name: str, time_limit: int = 0, **overrides) -> RwareConfig:
    m = _ID.match(str(name))
    if not m:
        raise ValueError(f"unsupported RWARE id {name!r}: expected [rware:]rware-{{tiny|small|medium|large}}-{{N}}ag[-easy|-hard]-v2")
    if m["v"] != "2":
        raise ValueError(f"{name!r}: only the v2 RWARE ids (rware 2.x, gymnasium) are implemented on the GPU path")
    if m["size"] not in SIZES:
        raise ValueError(f"{name!r}: unknown warehouse size {m['size']!r} (known: {', '.join(SIZES)})")
    n = int(m["n"])
    if not 1 <= n <= MAX_AGENTS:
        raise ValueError(f"{name!r}: {n} agents; the GPU path runs 1..{MAX_AGENTS} agents per warehouse")
    obs_type = str(overrides.pop("observation_type", "flattened")).lower()
    if obs_type not in ("flattened", "observationtype.flattened"):
        raise ValueError(f"{name!r}: observation_type {obs_type!r} is not implemented (the GPU path builds the flattened observation only)")
    if int(overrides.pop("msg_bits", 0) or 0) != 0:
        raise ValueError(f"{name!r}: msg_bits > 0 (agent messages) is not implemented on the GPU path")
    reward_type = str(overrides.pop("reward_type", "individual")).lower()
    if reward_type not in ("individual", "rewardtype.individual"):
        raise ValueError(f"{name!r}: reward_type {reward_type!r} is not implemented (the GPU path pays individual rewards only)")
    rows, cols = SIZES[m["size"]]
    cfg = RwareConfig(shelf_rows=rows, shelf_columns=cols, n_agents=n, request_queue_size=int(n * DIFFICULTY[m["diff"]]),
                      max_inactivity_steps=int(MAX_INACTIVITY_STEPS or 0), time_limit=int(time_limit or 0))
    for k, val in overrides.items():
        if k not in _OVERRIDES:
            raise TypeError(f"unknown RWARE option {k!r} (known: {', '.join(_OVERRIDES)})")
        setattr(cfg, k, int(val or 0))
    return cfg


class NativeRware(NativeEnv):
    """E warehouses on one device, the same surface as codebase_b200.lbf.NativeLbf."""

    PREFIX = "rware"

    def _env_fields(self):
        return (("shelves", torch.uint8, (self.cfg.rows * self.cfg.cols,)), ("agents", torch.uint8, (self.N, 4)), ("requested", torch.int32, (8,)),
                ("step", torch.int32, ()), ("inactive", torch.int32, ()))

    def set_state(self, shelves: torch.Tensor, agents: torch.Tensor, requested: torch.Tensor, step: torch.Tensor, inactive: torch.Tensor):
        """shelves uint8 [E][rows*cols] (shelf id at its current cell, 0 none), agents uint8 [E][N][4] = (x, y, dir, carried shelf id),
        requested uint32 [E][8] (bit k of the 256-bit mask: shelf k is requested), step / inactive int32 [E]."""
        self._set_state(shelves, agents, requested, step, inactive)

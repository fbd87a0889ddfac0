"""Low-level Python handle over the native repeated matrix games (marl_matrix_* entry points of libmarlb200.so).

All arrays are torch CUDA tensors; nothing here computes on the CPU.  Env ids follow the registration of the ``matrixgames`` package, the
companion of the MARL book: ``[matrixgames:]climbing[-nostate]-v0`` and ``[matrixgames:]penalty-{k}[-nostate]-v0`` for k in 0, 25, 50, 75,
100.  The payoffs and constructor defaults are recalled, not checked against the package (DESIGN.md Appendix C); every recalled value is a
named constant below, so a correction is a one-line change.
"""
from __future__ import annotations

import ctypes as C
import re
from dataclasses import dataclass, field

import numpy as np
import torch

from . import _native as nat
from .native_env import NativeEnv

_ID = re.compile(r"^(?:matrixgames:)?(?P<game>[a-z]+(?:-\d+)?)(?P<nostate>-nostate)?-v(?P<v>\d+)$")

CLIMBING = ((11, -30, 0), (-30, 7, 6), (0, 0, 5))   # (recalled)
PENALTY_KS = (0, 25, 50, 75, 100)                    # (recalled) the registered penalty-k ids
EP_LENGTH = 25                                       # (recalled) MatrixGame's ep_length default
VERSION = "0"                                        # (recalled) every registered id is -v0


def penalty(k: int) -> tuple:
    """The penalty game's payoff with penalty k."""
    return ((-k, 0, 10), (0, 2, 0), (10, 0, -k))   # (recalled)


GAMES = {"climbing": CLIMBING, **{f"penalty-{k}": penalty(k) for k in PENALTY_KS}}
MAX_ACTIONS = 8           # per player, on the GPU path
MAX_ENTRIES = 65536       # A^N payoff entries, on the GPU path
MAX_AGENTS = nat.MAX_AGENTS
_OVERRIDES = ("payoff_matrix", "ep_length", "last_action_state")


@dataclass
class MatrixConfig:
    payoff: np.ndarray = field(default_factory=lambda: np.asarray(CLIMBING, np.float64))   # float64, N dims of A entries each
    ep_length: int = EP_LENGTH
    last_action_state: int = 1     # 0: the -nostate ids
    time_limit: int = 0            # TimeLimit wrapper, env.time_limit; 0 = absent
    cooperative_reward: int = 0    # CooperativeReward wrapper
    observe_id: int = 0            # ObserveID wrapper
    standardise_rewards: int = 0   # StandardiseReward wrapper

    @property
    def n_agents(self) -> int:
        return int(self.payoff.ndim)

    @property
    def n_actions(self) -> int:
        return int(self.payoff.shape[0])

    @property
    def obs_dim(self) -> int:
        return (self.n_agents * self.n_actions if self.last_action_state else 1) + (self.n_agents if self.observe_id else 0)

    @property
    def obs_bounds(self) -> tuple[float, float]:
        """Observation-space bounds: one-hot features."""
        return 0.0, 1.0

    def to_native(self) -> nat.MatrixCfg:
        table = np.ascontiguousarray(self.payoff, np.float64)
        s = nat.MatrixCfg(self.n_agents, self.n_actions, table.ctypes.data_as(C.POINTER(C.c_double)), int(self.ep_length), int(self.last_action_state),
                          int(self.time_limit), int(self.cooperative_reward), int(self.observe_id), int(self.standardise_rewards))
        s._table = table   # the struct points into it
        return s


def is_matrix_id(name: str) -> bool:
    """A `matrixgames:` id, or a bare id naming one of the registered games."""
    name = str(name)
    if name.startswith("matrixgames:"):
        return True
    m = _ID.match(name)
    return bool(m) and m["game"] in GAMES


def payoff_table(payoff) -> np.ndarray:
    """The payoff as float64 [A]*N; ValueError for a table the GPU path does not run."""
    try:
        p = np.array(payoff, dtype=np.float64)
    except (ValueError, TypeError) as e:
        raise ValueError(f"payoff_matrix must be a rectangular array of numbers: {e}") from None
    if p.ndim < 1 or p.size == 0:
        raise ValueError(f"payoff_matrix must have one dimension per player and at least one action, got shape {p.shape}")
    if len(set(p.shape)) != 1:
        raise ValueError(f"payoff_matrix of shape {p.shape}: the GPU path needs the same number of actions for every player")
    if p.ndim > MAX_AGENTS:
        raise ValueError(f"payoff_matrix has {p.ndim} players; the GPU path runs 1..{MAX_AGENTS}")
    if p.shape[0] > MAX_ACTIONS:
        raise ValueError(f"payoff_matrix has {p.shape[0]} actions per player; the GPU path runs 1..{MAX_ACTIONS}")
    if p.size > MAX_ENTRIES:
        raise ValueError(f"payoff_matrix has {p.size} entries; the GPU path holds at most {MAX_ENTRIES}")
    return p


def parse_matrix_id(name: str, time_limit: int = 0, **overrides) -> MatrixConfig:
    m = _ID.match(str(name))
    if not m or m["game"] not in GAMES:
        raise ValueError(f"unsupported matrix game id {name!r}: expected [matrixgames:]{{climbing|penalty-{{{'|'.join(map(str, PENALTY_KS))}}}}}"
                         "[-nostate]-v0")
    if m["v"] != VERSION:
        raise ValueError(f"{name!r}: only the v{VERSION} matrix game ids are registered")
    for k in overrides:
        if k not in _OVERRIDES:
            raise TypeError(f"unknown matrix game option {k!r} (known: {', '.join(_OVERRIDES)})")
    cfg = MatrixConfig(payoff=payoff_table(overrides.get("payoff_matrix", GAMES[m["game"]])), time_limit=int(time_limit or 0),
                       last_action_state=int(not m["nostate"]))
    if "ep_length" in overrides:
        cfg.ep_length = int(overrides["ep_length"])
        if cfg.ep_length < 1:
            raise ValueError(f"{name!r}: ep_length must be >= 1, got {cfg.ep_length}")
    if "last_action_state" in overrides:
        cfg.last_action_state = int(bool(overrides["last_action_state"]))
    return cfg


class NativeMatrix(NativeEnv):
    """E matrix games on one device, the same surface as codebase_b200.lbf.NativeLbf."""

    PREFIX = "matrix"

    def _env_fields(self):
        return (("last_action", torch.int8, (self.N,)), ("step", torch.int32, ()))

    def set_state(self, last_action: torch.Tensor, step: torch.Tensor):
        """last_action int8 [E][N] (each player's previous action, -1: none), step int32 [E]."""
        self._set_state(last_action, step)

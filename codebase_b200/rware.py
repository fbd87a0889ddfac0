"""Low-level Python handle over the native multi-robot warehouse env (marl_rware_* entry points of libmarlb200.so).

All arrays are torch CUDA tensors; nothing here computes on the CPU.  Env ids follow the third-party ``rware`` 2.x registration
(gymnasium) the reference's README recommends: ``[rware:]rware-{size}-{N}ag[-easy|-hard]-v2``.  The constructor arguments of those ids
are recalled, not checked against the package (DESIGN.md Appendix B); every recalled value is a named constant below or a config field,
so a correction is a one-line change.
"""
from __future__ import annotations

import ctypes as C
import re
from dataclasses import dataclass, asdict

import torch

from . import _native as nat

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


class NativeRware:
    """E warehouses on one device, the same surface as codebase_b200.lbf.NativeLbf (reset, step, rollout_step, set_state, get_state)."""

    def __init__(self, cfg: RwareConfig, n_envs: int, seed: int, env_gid0: int = 0, device: int | None = None):
        if not torch.cuda.is_available():
            raise nat.NativeError("codebase_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        self.cfg, self.E, self.seed, self.gid0 = cfg, int(n_envs), int(seed), int(env_gid0)
        self.device_index = torch.cuda.current_device() if device is None else int(device)
        self.device = torch.device("cuda", self.device_index)
        self.N, self.D, self.A = cfg.n_agents, cfg.obs_dim, cfg.n_actions
        self._ncfg = cfg.to_native()
        self._h = C.c_void_p()
        self._lib = nat.lib()
        nat.check(self._lib.marl_rware_create(C.byref(self._ncfg), C.c_int32(self.E), C.c_uint64(self.seed & (2**64 - 1)), C.c_uint32(self.gid0),
                                              C.c_int32(self.device_index), C.byref(self._h)), "marl_rware_create")
        dev = self.device
        self.obs = torch.zeros(self.E, self.N, self.D, dtype=torch.float32, device=dev)
        self.rew = torch.zeros(self.E, self.N, dtype=torch.float32, device=dev)
        self.done = torch.zeros(self.E, dtype=torch.uint8, device=dev)
        self.trunc = torch.zeros(self.E, dtype=torch.uint8, device=dev)
        self.final_ret = torch.zeros(self.E, self.N, dtype=torch.float32, device=dev)
        self.final_len = torch.zeros(self.E, dtype=torch.int32, device=dev)
        self.actions = torch.zeros(self.E, self.N, dtype=torch.int32, device=dev)

    def close(self):
        if self._h:
            self._lib.marl_rware_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self, mask: torch.Tensor | None = None, traj=None, slot0: int = 0) -> torch.Tensor:
        nat.check(self._lib.marl_rware_reset(self._h, nat.ptr(mask), nat.ptr(self.obs), traj.ref() if traj else None, C.c_int32(slot0), nat.stream_ptr()),
                  "marl_rware_reset")
        return self.obs

    def step(self, actions: torch.Tensor, autoreset: bool = False):
        assert actions.dtype == torch.int32 and tuple(actions.shape) == (self.E, self.N)
        nat.check(self._lib.marl_rware_step(self._h, nat.ptr(actions), nat.ptr(self.obs), nat.ptr(self.rew), nat.ptr(self.done), nat.ptr(self.trunc),
                                            nat.ptr(self.final_ret), nat.ptr(self.final_len), C.c_int32(int(autoreset)), nat.stream_ptr()), "marl_rware_step")
        return self.obs, self.rew, self.done, self.trunc

    def rollout_step(self, values: torch.Tensor, policy: int, epsilon: float = 0.0, traj=None, slot0: int = 0,
                     use_proper_termination: bool = False, autoreset: bool = False, clear_stale: bool = False):
        """Fused categorical sampling on logits (policy 2) + transition + trajectory write; policy 1 (epsilon-greedy) is refused."""
        assert values.dtype == torch.float32 and values.shape[0] == self.E and values.shape[1] == self.N
        args = nat.RolloutArgs(policy, float(epsilon), int(values.shape[2]), int(use_proper_termination), int(autoreset), int(clear_stale), int(slot0))
        nat.check(self._lib.marl_rware_rollout_step(self._h, nat.ptr(values), C.byref(args), traj.ref() if traj else None, nat.ptr(self.obs), nat.ptr(self.rew),
                                                    nat.ptr(self.done), nat.ptr(self.trunc), nat.ptr(self.final_ret), nat.ptr(self.final_len),
                                                    nat.ptr(self.actions), nat.stream_ptr()), "marl_rware_rollout_step")
        return self.obs, self.rew, self.done, self.trunc

    def set_state(self, shelves: torch.Tensor, agents: torch.Tensor, requested: torch.Tensor, step: torch.Tensor, inactive: torch.Tensor):
        """shelves uint8 [E][rows*cols] (shelf id at its current cell, 0 none), agents uint8 [E][N][4] = (x, y, dir, carried shelf id),
        requested uint32 [E][8] (bit k of the 256-bit mask: shelf k is requested), step / inactive int32 [E]."""
        f = shelves.to(self.device, torch.uint8).contiguous().view(self.E, -1)
        a = agents.to(self.device, torch.uint8).contiguous().view(self.E, self.N, 4)
        q = requested.to(self.device, torch.int32).contiguous().view(self.E, 8)
        s = step.to(self.device, torch.int32).contiguous()
        i = inactive.to(self.device, torch.int32).contiguous()
        nat.check(self._lib.marl_rware_set_state(self._h, nat.ptr(f), nat.ptr(a), nat.ptr(q), nat.ptr(s), nat.ptr(i), nat.stream_ptr()), "marl_rware_set_state")
        torch.cuda.current_stream().synchronize()  # temporaries

    def get_state(self) -> dict:
        dev, E, N = self.device, self.E, self.N
        out = dict(shelves=torch.empty(E, self.cfg.rows * self.cfg.cols, dtype=torch.uint8, device=dev),
                   agents=torch.empty(E, N, 4, dtype=torch.uint8, device=dev), requested=torch.empty(E, 8, dtype=torch.int32, device=dev),
                   step=torch.empty(E, dtype=torch.int32, device=dev), inactive=torch.empty(E, dtype=torch.int32, device=dev),
                   ep_return=torch.empty(E, N, dtype=torch.float32, device=dev), ep_len=torch.empty(E, dtype=torch.int32, device=dev),
                   episode_idx=torch.empty(E, dtype=torch.int32, device=dev), active=torch.empty(E, dtype=torch.uint8, device=dev))
        keys = ("shelves", "agents", "requested", "step", "inactive", "ep_return", "ep_len", "episode_idx", "active")
        nat.check(self._lib.marl_rware_get_state(self._h, *[nat.ptr(out[k]) for k in keys], nat.stream_ptr()), "marl_rware_get_state")
        return out

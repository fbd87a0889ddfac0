"""Low-level Python handle over the native LBF env (marl_lbf_* entry points of libmarlb200.so).

All arrays are torch CUDA tensors; nothing here computes on the CPU.  Env ids follow the third-party
``lbforaging`` registration the reference passes to ``gym.make`` (marlbase/utils/envs.py:90-92,
README.md:80-85): ``[lbforaging:]Foraging[-grid][-2s]-{s}x{s}-{p}p-{f}f[-coop][-pen]-v{1,2,3}``.
"""
from __future__ import annotations

import ctypes as C
import re
from dataclasses import dataclass, asdict

import torch

from . import _native as nat

_ID = re.compile(r"^(?:lbforaging:)?Foraging(?P<grid>-grid)?(?P<po>-2s)?-(?P<s>\d+)x(?P<s2>\d+)-(?P<p>\d+)p-(?P<f>\d+)f(?P<coop>-coop)?(?P<pen>-pen)?-v(?P<v>\d+)$")


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

    @property
    def obs_dim(self) -> int:
        return 3 * self.max_num_food + 3 * self.n_agents + (self.n_agents if self.observe_id else 0)

    @property
    def n_actions(self) -> int:
        return 6

    def to_native(self) -> nat.LbfCfg:
        return nat.LbfCfg(**asdict(self))


def parse_env_id(name: str, time_limit: int = 0, **overrides) -> LbfConfig:
    m = _ID.match(name)
    if not m:
        raise ValueError(f"unsupported environment id {name!r}: the GPU path implements Level-Based Foraging ids only")
    if m["grid"]:
        raise ValueError("grid observations (Foraging-grid-*) are not implemented on the GPU path")
    s, s2, p, f, v = int(m["s"]), int(m["s2"]), int(m["p"]), int(m["f"]), int(m["v"])
    cfg = LbfConfig(rows=s, cols=s2, n_agents=p, max_num_food=f, sight=2 if m["po"] else s,
                    max_player_level=2 if v >= 3 else 3, force_coop=int(bool(m["coop"])),
                    penalty=0.1 if m["pen"] else 0.0, time_limit=int(time_limit or 0))
    for k, val in overrides.items():
        if not hasattr(cfg, k):
            raise TypeError(f"unknown LBF option {k!r}")
        setattr(cfg, k, val)
    return cfg


class TrajStore:
    """Episode-major trajectory store on the device: replay ring (marlbase/dqn/train.py:19-124) or on-policy batch
    (marlbase/ac/train.py:36-52)."""

    def __init__(self, capacity: int, n_agents: int, T: int, obs_dim: int, device):
        self.capacity, self.N, self.T, self.D = capacity, n_agents, T, obs_dim
        self.obs = torch.zeros(capacity, n_agents, T + 1, obs_dim, dtype=torch.float32, device=device)
        self.act = torch.zeros(capacity, n_agents, T, dtype=torch.int32, device=device)
        self.rew = torch.zeros(capacity, n_agents, T, dtype=torch.float32, device=device)
        self.done = torch.zeros(capacity, T + 1, dtype=torch.uint8, device=device)
        self.filled = torch.zeros(capacity, T, dtype=torch.uint8, device=device)
        self.view = nat.TrajView(nat.ptr(self.obs), nat.ptr(self.act), nat.ptr(self.rew), nat.ptr(self.done), nat.ptr(self.filled),
                                 capacity, n_agents, T, obs_dim)

    def ref(self):
        return C.byref(self.view)


class NativeLbf:
    def __init__(self, cfg: LbfConfig, n_envs: int, seed: int, env_gid0: int = 0, device: int | None = None):
        if not torch.cuda.is_available():
            raise nat.NativeError("codebase_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        self.cfg, self.E, self.seed, self.gid0 = cfg, int(n_envs), int(seed), int(env_gid0)
        self.device_index = torch.cuda.current_device() if device is None else int(device)
        self.device = torch.device("cuda", self.device_index)
        self.N, self.D, self.A = cfg.n_agents, cfg.obs_dim, cfg.n_actions
        self._ncfg = cfg.to_native()
        self._h = C.c_void_p()
        self._lib = nat.lib()
        nat.check(self._lib.marl_lbf_create(C.byref(self._ncfg), C.c_int32(self.E), C.c_uint64(self.seed & (2**64 - 1)), C.c_uint32(self.gid0),
                                            C.c_int32(self.device_index), C.byref(self._h)), "marl_lbf_create")
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
            self._lib.marl_lbf_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self, mask: torch.Tensor | None = None, traj: TrajStore | None = None, slot0: int = 0) -> torch.Tensor:
        nat.check(self._lib.marl_lbf_reset(self._h, nat.ptr(mask), nat.ptr(self.obs), traj.ref() if traj else None, C.c_int32(slot0), nat.stream_ptr()),
                  "marl_lbf_reset")
        return self.obs

    def step(self, actions: torch.Tensor, autoreset: bool = False):
        assert actions.dtype == torch.int32 and tuple(actions.shape) == (self.E, self.N)
        nat.check(self._lib.marl_lbf_step(self._h, nat.ptr(actions), nat.ptr(self.obs), nat.ptr(self.rew), nat.ptr(self.done), nat.ptr(self.trunc),
                                          nat.ptr(self.final_ret), nat.ptr(self.final_len), C.c_int32(int(autoreset)), nat.stream_ptr()), "marl_lbf_step")
        return self.obs, self.rew, self.done, self.trunc

    def rollout_step(self, values: torch.Tensor, policy: int, epsilon: float = 0.0, traj: TrajStore | None = None, slot0: int = 0,
                     use_proper_termination: bool = False, autoreset: bool = False, clear_stale: bool = False):
        """Fused action selection (1 = eps-greedy on Q-values, 2 = categorical on logits) + transition + trajectory write."""
        assert values.dtype == torch.float32 and values.shape[0] == self.E and values.shape[1] == self.N
        args = nat.RolloutArgs(policy, float(epsilon), int(values.shape[2]), int(use_proper_termination), int(autoreset), int(clear_stale), int(slot0))
        nat.check(self._lib.marl_lbf_rollout_step(self._h, nat.ptr(values), C.byref(args), traj.ref() if traj else None, nat.ptr(self.obs), nat.ptr(self.rew),
                                                  nat.ptr(self.done), nat.ptr(self.trunc), nat.ptr(self.final_ret), nat.ptr(self.final_len), nat.ptr(self.actions),
                                                  nat.stream_ptr()), "marl_lbf_rollout_step")
        return self.obs, self.rew, self.done, self.trunc

    def set_state(self, field: torch.Tensor, players: torch.Tensor, step: torch.Tensor):
        f = field.to(self.device, torch.int8).contiguous().view(self.E, -1)
        p = players.to(self.device, torch.int8).contiguous().view(self.E, self.N, 4)
        s = step.to(self.device, torch.int32).contiguous()
        nat.check(self._lib.marl_lbf_set_state(self._h, nat.ptr(f), nat.ptr(p), nat.ptr(s), nat.stream_ptr()), "marl_lbf_set_state")
        torch.cuda.current_stream().synchronize()  # f/p/s are temporaries

    def get_state(self) -> dict:
        dev, E, N = self.device, self.E, self.N
        out = dict(field=torch.empty(E, self.cfg.rows * self.cfg.cols, dtype=torch.int8, device=dev),
                   players=torch.empty(E, N, 4, dtype=torch.int8, device=dev), step=torch.empty(E, dtype=torch.int32, device=dev),
                   food_spawned=torch.empty(E, dtype=torch.int32, device=dev), ep_return=torch.empty(E, N, dtype=torch.float32, device=dev),
                   ep_len=torch.empty(E, dtype=torch.int32, device=dev), episode_idx=torch.empty(E, dtype=torch.int32, device=dev),
                   active=torch.empty(E, dtype=torch.uint8, device=dev))
        nat.check(self._lib.marl_lbf_get_state(self._h, *[nat.ptr(out[k]) for k in ("field", "players", "step", "food_spawned", "ep_return", "ep_len", "episode_idx", "active")],
                                               nat.stream_ptr()), "marl_lbf_get_state")
        return out

"""Python handle layer shared by the native envs (marl_lbf_* and marl_rware_* entry points of libmarlb200.so), and the trajectory store
their rollout steps and every learner use.

All arrays are torch CUDA tensors; nothing here computes on the CPU.
"""
from __future__ import annotations

import ctypes as C

import torch

from . import _native as nat


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


class NativeEnv:
    """E envs of one kind on one device, driven through the C entry points marl_<PREFIX>_*.

    A subclass sets PREFIX and implements `_env_fields`: its own part of the state as (name, dtype, per-env shape), in the argument order of
    marl_<PREFIX>_get_state, which continues with the episode record of every env kind.  Its `set_state` passes the leading fields that
    marl_<PREFIX>_set_state takes to `_set_state`."""

    PREFIX = ""

    def __init__(self, cfg, n_envs: int, seed: int, env_gid0: int = 0, device: int | None = None):
        if not torch.cuda.is_available():
            raise nat.NativeError("codebase_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        self.cfg, self.E, self.seed, self.gid0 = cfg, int(n_envs), int(seed), int(env_gid0)
        self.device_index = torch.cuda.current_device() if device is None else int(device)
        self.device = torch.device("cuda", self.device_index)
        self.N, self.D, self.A = cfg.n_agents, cfg.obs_dim, cfg.n_actions
        self._ncfg = cfg.to_native()
        self._h = C.c_void_p()
        lib = nat.lib()
        # resolved once: the rollout loop crosses into the library on every env step
        (self._c_create, self._c_destroy, self._c_reset, self._c_step, self._c_rollout_step, self._c_set_state, self._c_get_state) = (
            getattr(lib, f"marl_{self.PREFIX}_{name}") for name in ("create", "destroy", "reset", "step", "rollout_step", "set_state", "get_state"))
        nat.check(self._c_create(C.byref(self._ncfg), C.c_int32(self.E), C.c_uint64(self.seed & (2**64 - 1)), C.c_uint32(self.gid0),
                               C.c_int32(self.device_index), C.byref(self._h)), self._c_create.__name__)
        dev = self.device
        self.obs = torch.zeros(self.E, self.N, self.D, dtype=torch.float32, device=dev)
        self.rew = torch.zeros(self.E, self.N, dtype=torch.float32, device=dev)
        self.done = torch.zeros(self.E, dtype=torch.uint8, device=dev)
        self.trunc = torch.zeros(self.E, dtype=torch.uint8, device=dev)
        self.final_ret = torch.zeros(self.E, self.N, dtype=torch.float32, device=dev)
        self.final_len = torch.zeros(self.E, dtype=torch.int32, device=dev)
        self.actions = torch.zeros(self.E, self.N, dtype=torch.int32, device=dev)
        self._c_render = getattr(lib, f"marl_{self.PREFIX}_render")
        h, w = C.c_int32(), C.c_int32()
        fs = getattr(lib, f"marl_{self.PREFIX}_frame_shape")
        nat.check(fs(C.byref(self._ncfg), C.byref(h), C.byref(w)), fs.__name__)
        self.frame_shape = (h.value, w.value, 3)

    def render(self, env_first: int = 0, n: int = 1, out: torch.Tensor | None = None) -> torch.Tensor:
        """RGB frames of envs [env_first, env_first + n), one launch: device uint8 [n, H, W, 3] (`out`, or a new tensor); H, W, 3 = frame_shape."""
        if out is None:
            out = torch.empty(int(n), *self.frame_shape, dtype=torch.uint8, device=self.device)
        assert out.dtype == torch.uint8 and tuple(out.shape) == (int(n), *self.frame_shape), "render: out must be uint8 [n, H, W, 3]"
        nat.check(self._c_render(self._h, C.c_int32(env_first), C.c_int32(n), nat.ptr(out), nat.stream_ptr()), self._c_render.__name__)
        return out

    def close(self):
        if self._h:
            self._c_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self, mask: torch.Tensor | None = None, traj: TrajStore | None = None, slot0: int = 0) -> torch.Tensor:
        nat.check(self._c_reset(self._h, nat.ptr(mask), nat.ptr(self.obs), traj.ref() if traj else None, C.c_int32(slot0), nat.stream_ptr()),
                  self._c_reset.__name__)
        return self.obs

    def step(self, actions: torch.Tensor, autoreset: bool = False):
        assert actions.dtype == torch.int32 and tuple(actions.shape) == (self.E, self.N)
        nat.check(self._c_step(self._h, nat.ptr(actions), nat.ptr(self.obs), nat.ptr(self.rew), nat.ptr(self.done), nat.ptr(self.trunc),
                             nat.ptr(self.final_ret), nat.ptr(self.final_len), C.c_int32(int(autoreset)), nat.stream_ptr()), self._c_step.__name__)
        return self.obs, self.rew, self.done, self.trunc

    def rollout_step(self, values: torch.Tensor, policy: int, epsilon: float = 0.0, traj: TrajStore | None = None, slot0: int = 0,
                     use_proper_termination: bool = False, autoreset: bool = False, clear_stale: bool = False):
        """Fused action selection (1 = eps-greedy on Q-values, 2 = categorical on logits) + transition + trajectory write."""
        assert values.dtype == torch.float32 and values.shape[0] == self.E and values.shape[1] == self.N
        args = nat.RolloutArgs(policy, float(epsilon), int(values.shape[2]), int(use_proper_termination), int(autoreset), int(clear_stale), int(slot0))
        nat.check(self._c_rollout_step(self._h, nat.ptr(values), C.byref(args), traj.ref() if traj else None, nat.ptr(self.obs), nat.ptr(self.rew),
                                     nat.ptr(self.done), nat.ptr(self.trunc), nat.ptr(self.final_ret), nat.ptr(self.final_len), nat.ptr(self.actions),
                                     nat.stream_ptr()), self._c_rollout_step.__name__)
        return self.obs, self.rew, self.done, self.trunc

    def _env_fields(self) -> tuple:
        raise NotImplementedError

    def _state_fields(self) -> tuple:
        return self._env_fields() + (("ep_return", torch.float32, (self.N,)), ("ep_len", torch.int32, ()), ("episode_idx", torch.int32, ()),
                                     ("active", torch.uint8, ()))

    def _set_state(self, *values: torch.Tensor):
        tmp = [v.to(self.device, dtype).contiguous().view(self.E, *shape) for v, (_, dtype, shape) in zip(values, self._state_fields())]
        nat.check(self._c_set_state(self._h, *[nat.ptr(t) for t in tmp], nat.stream_ptr()), self._c_set_state.__name__)
        torch.cuda.current_stream().synchronize()  # tmp are temporaries

    def get_state(self) -> dict:
        out = {name: torch.empty(self.E, *shape, dtype=dtype, device=self.device) for name, dtype, shape in self._state_fields()}
        nat.check(self._c_get_state(self._h, *[nat.ptr(t) for t in out.values()], nat.stream_ptr()), self._c_get_state.__name__)
        return out

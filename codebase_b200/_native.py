"""ctypes binding of libmarlb200.so -- the only route from Python into the CUDA hot path.

There is no CPU fallback: if the library is missing, cannot be loaded, or an entry point reports an error,
a :class:`NativeError` is raised.  torch is used for device memory and streams only (plumbing).
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("MARL_B200_SO") or os.path.join(_HERE, "csrc", "libmarlb200.so")   # MARL_B200_SO: a profiling build of the same library
_lib = None


class NativeError(RuntimeError):
    pass


class LbfCfg(C.Structure):
    _fields_ = [
        ("rows", C.c_int32), ("cols", C.c_int32), ("n_agents", C.c_int32), ("max_num_food", C.c_int32),
        ("sight", C.c_int32), ("min_player_level", C.c_int32), ("max_player_level", C.c_int32),
        ("min_food_level", C.c_int32), ("max_food_level", C.c_int32), ("max_episode_steps", C.c_int32),
        ("time_limit", C.c_int32), ("force_coop", C.c_int32), ("normalize_reward", C.c_int32),
        ("cooperative_reward", C.c_int32), ("penalty", C.c_double), ("observe_id", C.c_int32), ("standardise_rewards", C.c_int32), ("upstream_reset", C.c_int32),
        ("grid_observation", C.c_int32),
    ]


class RwareCfg(C.Structure):
    _fields_ = [
        ("shelf_rows", C.c_int32), ("shelf_columns", C.c_int32), ("column_height", C.c_int32), ("n_agents", C.c_int32),
        ("request_queue_size", C.c_int32), ("max_steps", C.c_int32), ("max_inactivity_steps", C.c_int32), ("sensor_range", C.c_int32),
        ("time_limit", C.c_int32), ("cooperative_reward", C.c_int32), ("observe_id", C.c_int32), ("standardise_rewards", C.c_int32),
    ]


class MatrixCfg(C.Structure):
    _fields_ = [
        ("n_agents", C.c_int32), ("n_actions", C.c_int32), ("payoff", C.POINTER(C.c_double)), ("ep_length", C.c_int32),
        ("last_action_state", C.c_int32), ("time_limit", C.c_int32), ("cooperative_reward", C.c_int32), ("observe_id", C.c_int32),
        ("standardise_rewards", C.c_int32),
    ]


class TrajView(C.Structure):
    _fields_ = [
        ("obs", C.c_void_p), ("act", C.c_void_p), ("rew", C.c_void_p), ("done", C.c_void_p), ("filled", C.c_void_p),
        ("capacity", C.c_int32), ("n_agents", C.c_int32), ("T", C.c_int32), ("obs_dim", C.c_int32),
    ]


class RolloutArgs(C.Structure):
    _fields_ = [
        ("policy", C.c_int32), ("epsilon", C.c_float), ("n_actions", C.c_int32), ("use_proper_termination", C.c_int32),
        ("autoreset", C.c_int32), ("clear_stale", C.c_int32), ("slot0", C.c_int32),
    ]


MAX_AGENTS = 32   # MARL_MAX_AGENTS (include/marl_b200.h): the length of marl_mlp_cfg.agent_net


class MlpCfg(C.Structure):
    _fields_ = [("n_agents", C.c_int32), ("n_nets", C.c_int32), ("agent_net", C.c_int32 * MAX_AGENTS), ("in_dim", C.c_int32),
                ("hidden", C.c_int32), ("out_dim", C.c_int32)]


class DqnHP(C.Structure):
    _fields_ = [("lr", C.c_float), ("gamma", C.c_float), ("grad_clip", C.c_float), ("double_q", C.c_int32),
                ("target_update_interval_or_tau", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float), ("eps", C.c_float),
                ("mixer", C.c_int32)]


class A2cHP(C.Structure):
    _fields_ = [("lr", C.c_float), ("gamma", C.c_float), ("grad_clip", C.c_float), ("n_steps", C.c_int32), ("entropy_coef", C.c_float),
                ("value_loss_coef", C.c_float), ("target_update_interval_or_tau", C.c_float), ("beta1", C.c_float), ("beta2", C.c_float),
                ("eps", C.c_float)]


class Optimizer(C.Structure):
    _fields_ = [("kind", C.c_int32), ("beta1", C.c_double), ("beta2", C.c_double), ("alpha", C.c_double), ("eps", C.c_double),
                ("weight_decay", C.c_double)]


class _DevArray:
    """Zero-copy torch view of library-owned device memory through the CUDA array interface."""

    def __init__(self, ptr: int, n: int, typestr: str = "<f4"):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2}


def device_view(ptr: int, n: int, device, typestr: str = "<f4"):
    import torch

    return torch.as_tensor(_DevArray(ptr, n, typestr), device=device)


def lib():
    """Load libmarlb200.so; raise loudly when it is absent (run `python -c 'import __graft_entry__ as g; g.build()'`)."""
    global _lib
    if _lib is None:
        if not os.path.exists(SO_PATH):
            raise NativeError(f"{SO_PATH} is missing: build it with __graft_entry__.build(); there is no CPU fallback")
        try:
            _lib = C.CDLL(SO_PATH)
        except OSError as e:  # pragma: no cover
            raise NativeError(f"cannot load {SO_PATH}: {e}") from e
        _lib.marl_last_error.restype = C.c_char_p
        if _lib.marl_version() != 1:
            raise NativeError("libmarlb200.so ABI version mismatch")
    return _lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = lib().marl_last_error().decode("utf8", "replace")
        raise NativeError(f"{what} failed (rc={rc}): {msg}")


def ptr(t):
    """Device pointer of a torch tensor (or None)."""
    if t is None:
        return C.c_void_p(None)
    assert t.is_cuda and t.is_contiguous(), "native entry points take contiguous CUDA tensors"
    return C.c_void_p(t.data_ptr())


def stream_ptr():
    import torch

    return C.c_void_p(torch.cuda.current_stream().cuda_stream)

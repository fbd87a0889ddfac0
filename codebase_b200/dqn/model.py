"""IDQN / VDN learners on the GPU path -- drop-in for marlbase/dqn/model.py (QNetwork 14-196, VDNetwork 199-269).

Same constructor signature and Hydra `_target_` role (configs/algorithm/idqn.yaml:6-14, vdn.yaml:11-13), same
`state_dict()` key names (`critic.independent.{i}.network.{0,2,4}.{weight,bias}`, `target.…`; shared:
`critic.networks.{k}.…`) so checkpoints interchange with the reference's eval.py.  All arithmetic runs in
libmarlb200.so (marl_dqn_*); torch is used for parameter initialisation (nn.init on the host, once) and as the
owner of device buffers.  There is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import math
import numbers
import random
import types

import numpy as np
import torch

from .. import _native as nat
from .. import optimizers
from ..learner import MAX_AGENTS, NativeLearner, flat_to_state_dict, flatdim, hidden_width, init_flat_params, init_flat_rnn_params, mlp_shapes, rnn_shapes, \
    sharing_to_nets, state_dict_to_flat
from ..native_env import TrajStore


def td_lambda(cfg):
    """cfg.td_lambda: None (absent or null: the reference's one-step TD target) or the λ in [0, 1] of the TD(λ) target that replaces it.  Anything
    else raises ValueError here, before any native call."""
    lam = getattr(cfg, "td_lambda", None)
    if lam is None:
        return None
    if isinstance(lam, bool) or not isinstance(lam, numbers.Real):
        raise ValueError(f"algorithm.td_lambda must be null or a number in [0, 1], not {lam!r}")
    lam = float(lam)
    if not 0.0 <= lam <= 1.0:
        raise ValueError(f"algorithm.td_lambda must be in [0, 1], not {lam}")
    return lam


def huber_delta(cfg):
    """cfg.huber_delta: None (absent or null: the reference's squared TD error) or the finite delta > 0 of the Huber TD loss that replaces it.
    Anything else raises ValueError here, before any native call."""
    delta = getattr(cfg, "huber_delta", None)
    if delta is None:
        return None
    if isinstance(delta, bool) or not isinstance(delta, numbers.Real):
        raise ValueError(f"algorithm.huber_delta must be null or a finite number > 0, not {delta!r}")
    delta = float(delta)
    if not (math.isfinite(delta) and delta > 0.0):
        raise ValueError(f"algorithm.huber_delta must be a finite number > 0, not {delta}")
    return delta


class QNetwork(NativeLearner):
    mixer = 0
    _destroy = "marl_dqn_destroy"

    def __init__(self, obs_space, action_space, cfg, layers, parameter_sharing, use_rnn, use_orthogonal_init, device, max_batch=None, max_episode_length=None):
        self.td_lambda = td_lambda(cfg)
        self.huber_delta = huber_delta(cfg)
        self.use_rnn = bool(use_rnn)
        self.hidden = hidden_width(layers, "layers", self.use_rnn)
        self._open(obs_space, action_space, cfg, device)
        self._shapes = (rnn_shapes if self.use_rnn else mlp_shapes)(self.in_dim, self.n_actions, self.hidden)
        self.action_space = action_space
        self.agent_net = sharing_to_nets(parameter_sharing, self.n_agents)
        self.n_nets = max(self.agent_net) + 1
        self._kind = "independent" if not parameter_sharing else "networks"
        self.gamma, self.grad_clip, self.double_q = float(cfg.gamma), cfg.grad_clip, bool(cfg.double_q)
        self.target_update_interval_or_tau = float(cfg.target_update_interval_or_tau)
        self.max_batch = int(max_batch or getattr(cfg, "batch_size", 1024))
        self.max_T = int(max_episode_length or getattr(cfg, "max_episode_length", 0) or 500)
        mcfg = nat.MlpCfg(self.n_agents, self.n_nets, (C.c_int32 * MAX_AGENTS)(*self.agent_net), self.in_dim, self.hidden, self.n_actions)
        hp = nat.DqnHP(float(cfg.lr), self.gamma, float(self.grad_clip or 0.0), int(self.double_q), self.target_update_interval_or_tau,
                       0.9, 0.999, 1e-8, self.mixer)
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):
            create = self._lib.marl_dqn_create_rnn if self.use_rnn else self._lib.marl_dqn_create
            nat.check(create(C.byref(mcfg), C.byref(hp), C.c_int32(self.max_batch), C.c_int32(self.max_T), C.c_int32(self.device.index),
                             C.byref(self._h)), "marl_dqn_create_rnn" if self.use_rnn else "marl_dqn_create")
        optimizers.apply(self._lib, "marl_dqn_set_optimizer", self._h, self.optimizer_name)
        ptrs = [C.c_void_p() for _ in range(5)]
        n = C.c_int64()
        nat.check(self._lib.marl_dqn_param_ptrs(self._h, *[C.byref(p) for p in ptrs], C.byref(n)), "marl_dqn_param_ptrs")
        self.n_params = int(n.value)
        self.theta, self.theta_tgt, self.adam_m, self.adam_v = [nat.device_view(p.value, self.n_params, self.device) for p in ptrs[:4]]
        self.grad = nat.device_view(ptrs[4].value, self.n_params + 4, self.device)  # + (loss numerator, filled count, 2 spare)
        init = init_flat_rnn_params if self.use_rnn else init_flat_params
        self.theta.copy_(init(self.n_nets, self.in_dim, self.n_actions, use_orthogonal_init, self.hidden))
        self.params_changed()
        self.hard_update()
        self._metrics = torch.zeros(6, dtype=torch.float32, device=self.device)
        self._idx = torch.zeros(self.max_batch, dtype=torch.int32, device=self.device)
        self.standardise_returns = bool(getattr(cfg, "standardise_returns", False))   # dqn/model.py:82-84 (VDN: 221-222)
        if self.standardise_returns:
            nat.check(self._lib.marl_dqn_standardise_returns(self._h, C.c_int32(1)), "marl_dqn_standardise_returns")
        if self.td_lambda is not None:
            self.set_td_lambda(self.td_lambda)
        if self.huber_delta is not None:
            self.set_huber_delta(self.huber_delta)

    def set_td_lambda(self, lam):
        """TD(λ) targets of `lam` in [0, 1] in place of the one-step target from the next update on (DESIGN.md §4.4d); None: the one-step target again"""
        lam = td_lambda(types.SimpleNamespace(td_lambda=lam))
        nat.check(self._lib.marl_dqn_set_td_lambda(self._h, C.c_int32(lam is not None), C.c_float(0.0 if lam is None else lam)), "marl_dqn_set_td_lambda")
        self.td_lambda = lam

    def set_huber_delta(self, delta):
        """The Huber TD loss with `delta` (a finite number > 0) in place of the squared TD error from the next update on (DESIGN.md §4.4e); None:
        the squared error again"""
        delta = huber_delta(types.SimpleNamespace(huber_delta=delta))
        nat.check(self._lib.marl_dqn_set_huber_delta(self._h, C.c_int32(delta is not None), C.c_float(0.0 if delta is None else delta)),
                  "marl_dqn_set_huber_delta")
        self.huber_delta = delta

    def ret_ms(self):
        """(mean, var, count) of the RunningMeanStd over the TD targets (standardise_returns): one entry per agent; VDN, QMIX: per batch entry."""
        pm, pc, n = C.c_void_p(), C.c_void_p(), C.c_int32()
        nat.check(self._lib.marl_dqn_ret_ms_ptrs(self._h, C.byref(pm), C.byref(pc), C.byref(n)), "marl_dqn_ret_ms_ptrs")
        ms = nat.device_view(pm.value, 2 * n.value, self.device).cpu()
        return ms[: n.value], ms[n.value:], float(nat.device_view(pc.value, 1, self.device, "<f8").cpu()[0])

    def scratch(self, B, T):
        """(bootstrap values, TD targets, chosen Q, dLoss/dQ) of the last update's external TD head, each [C,B,T] (C = N for IDQN, 1 for VDN and
        QMIX; QMIX's dLoss/dQ is per agent, [N,B,T]) or None where the handle has no such buffer -- device views for tests."""
        ptrs = [C.c_void_p() for _ in range(4)]
        nat.check(self._lib.marl_dqn_scratch_ptrs(self._h, *[C.byref(p) for p in ptrs]), "marl_dqn_scratch_ptrs")
        cols = [1 if self.mixer else self.n_agents] * 3 + [1 if self.mixer == 1 else self.n_agents]
        return tuple(None if p.value is None else nat.device_view(p.value, c * B * T, self.device).view(c, B, T) for p, c in zip(ptrs, cols))

    # ---- reference API ------------------------------------------------------------------------------------------
    def init_hiddens(self, batch_size):
        return self._hiddens(self.use_rnn, batch_size, self.hidden)

    def q_values(self, obs: torch.Tensor, target: bool = False, out: torch.Tensor | None = None, h: torch.Tensor | None = None,
                 h_out: torch.Tensor | None = None):
        """Network pass of model.act (dqn/model.py:96-99) for E envs: obs f32[E,N,D] -> q f32[E,N,A].
        Recurrent networks take one step from h f32[E,N,H] (None: the zero state) and return (q, h_out); h_out must not be h."""
        E = obs.shape[0]
        if out is None:
            out = torch.empty(E, self.n_agents, self.n_actions, dtype=torch.float32, device=self.device)
        if not self.use_rnn:
            nat.check(self._lib.marl_dqn_forward(self._h, nat.ptr(obs), C.c_int32(E), C.c_int32(int(target)), nat.ptr(out), nat.stream_ptr()), "marl_dqn_forward")
            return out
        if h_out is None:
            h_out = torch.empty(E, self.n_agents, self.hidden, dtype=torch.float32, device=self.device)
        nat.check(self._lib.marl_dqn_forward_rnn(self._h, nat.ptr(obs), C.c_int32(E), C.c_int32(int(target)), nat.ptr(h), nat.ptr(h_out), nat.ptr(out),
                                                 nat.stream_ptr()), "marl_dqn_forward_rnn")
        return out, h_out

    def act(self, inputs, hiddens, epsilon, action_masks=None):
        """dqn/model.py:94-116 for API parity (single env or a stack of envs).  The training / evaluation loops use the fused
        marl_lbf_rollout_step instead, which draws exploration from the Philox stream inside the env kernel."""
        if action_masks is not None:
            raise NotImplementedError("action masks only exist for smaclite in the reference (out of scope)")
        obs = torch.as_tensor(np.stack([np.asarray(i, np.float32) for i in inputs], 0), device=self.device)
        obs = obs.view(self.n_agents, -1, self.in_dim).transpose(0, 1).contiguous()
        if self.use_rnn:   # hiddens: per agent (1, E, H) or None (dqn/model.py:99 carries them through the critic)
            q, h_out = self.q_values(obs, h=self._stack_hiddens(hiddens, self.hidden))
            hiddens = self._split_hiddens(h_out)
        else:
            q = self.q_values(obs)
        # the reference's stream: ONE `random.random()` per call decides the joint exploration (dqn/model.py:105), the random joint
        # action comes from Python's `random` as well (seed it with random.seed, as the reference's users do)
        if epsilon > random.random():
            actions = torch.tensor([[random.randrange(self.n_actions) for _ in range(self.n_agents)] for _ in range(obs.shape[0])])
        else:
            actions = q.argmax(-1).cpu()
        return (actions[0].tolist() if actions.shape[0] == 1 else actions.T.tolist()), hiddens

    def update_from_store(self, traj: TrajStore, idx: torch.Tensor):
        """QNetwork.update on episodes `idx` (int32 device tensor) of a device trajectory store."""
        nat.check(self._lib.marl_dqn_update(self._h, traj.ref(), nat.ptr(idx), C.c_int32(idx.numel()), nat.ptr(self._metrics), nat.stream_ptr()), "marl_dqn_update")
        return self._metrics

    def update_grads(self, traj: TrajStore, idx: torch.Tensor):
        nat.check(self._lib.marl_dqn_update_grads(self._h, traj.ref(), nat.ptr(idx), C.c_int32(idx.numel()), nat.stream_ptr()), "marl_dqn_update_grads")

    def update_apply(self):
        nat.check(self._lib.marl_dqn_update_apply(self._h, nat.ptr(self._metrics), nat.stream_ptr()), "marl_dqn_update_apply")
        return self._metrics

    def update_n(self, traj: TrajStore, batch_size: int, n_valid: int, seed: int, first_update_idx: int, n_updates: int):
        """`rb.sample(batch); model.update(batch)` n times on device (dqn/train.py:308-311)."""
        nat.check(self._lib.marl_dqn_update_n(self._h, traj.ref(), C.c_int32(batch_size), C.c_int32(n_valid), C.c_uint64(seed & (2**64 - 1)),
                                              C.c_uint64(first_update_idx), C.c_int32(n_updates), nat.ptr(self._metrics), nat.stream_ptr()), "marl_dqn_update_n")
        return self._metrics

    def exchanged_buffers(self):
        """What data-parallel ranks sum between update_grads and update_apply: [gradient sums | loss numerator | filled count | 2 spare]."""
        return [self.grad]

    def update_n_allreduce(self, traj: TrajStore, batch_size: int, n_valid: int, seed: int, first_update_idx: int, n_updates: int, all_reduce):
        """update_n's updates (same replay indices) in the two-call form: per update sample, update_grads, `all_reduce(exchanged_buffers())` (an
        in-place sum over ranks), update_apply.  Every rank then divides by the global filled count and applies the same step."""
        for u in range(n_updates):
            nat.check(self._lib.marl_replay_sample(C.c_uint64(seed & (2**64 - 1)), C.c_uint64(first_update_idx + u), C.c_int32(batch_size), C.c_int32(n_valid),
                                                   nat.ptr(self._idx), nat.stream_ptr()), "marl_replay_sample")
            self.update_grads(traj, self._idx[:batch_size])
            all_reduce(self.exchanged_buffers())
            self.update_apply()
        return self._metrics

    def update(self, batch):
        """Reference signature (dqn/model.py:165-174): `batch` is the reference's Batch namedtuple (obss (N,T+1,B,obs), actions
        (N,T,B), rewards (N,T,B), dones (T+1,B), filled (T,B)); converted to the device layout, then the native update."""
        obss = batch.obss
        N, T1, B, D = obss.shape
        store = TrajStore(B, N, T1 - 1, D, self.device)
        store.obs.copy_(obss.permute(2, 0, 1, 3))
        store.act.copy_(batch.actions.permute(2, 0, 1))
        store.rew.copy_(batch.rewards.permute(2, 0, 1))
        store.done.copy_(batch.dones.permute(1, 0))
        store.filled.copy_(batch.filled.permute(1, 0))
        idx = torch.arange(B, dtype=torch.int32, device=self.device)
        m = self.update_from_store(store, idx)
        return {"loss": float(m[0].item())}

    def timing(self, enable: bool):
        """CUDA-event timing of the training kernel: timing(True) starts, timing(False) -> (total_ms, launches)."""
        ms, n = C.c_float(), C.c_int32()
        nat.check(self._lib.marl_dqn_timing(self._h, C.c_int32(int(enable)), C.byref(ms), C.byref(n)), "marl_dqn_timing")
        return float(ms.value), int(n.value)

    peers_attached = False

    def attach_peers(self, group=None):
        """Several ranks, one process per GPU: exchange CUDA IPC handles through torch.distributed and let `update` / `update_n` sum
        the gradients of all ranks over NVLink peer memory inside the fused reduce + Adam kernel (no all-reduce call per update).
        MLP and recurrent agent networks whose parameters fit one wave of the fused tail; QMIX's mixer gradient travels in the same exchange.
        Every rank makes the same collective calls whatever fails where, and either every rank returns or every rank raises NativeError (a rank
        that did attach keeps working with the two-call form: update_grads, an all-reduce, update_apply)."""
        import torch.distributed as dist

        world, rank = dist.get_world_size(group), dist.get_rank(group)
        mine, err = (C.c_ubyte * 64)(), None
        try:
            nat.check(self._lib.marl_dqn_peer_handle(self._h, mine), "marl_dqn_peer_handle")
        except nat.NativeError as e:
            err = str(e)
        handles = [None] * world
        dist.all_gather_object(handles, bytes(mine) if err is None else None, group=group)
        if err is None:
            if any(h is None for h in handles):
                err = "a peer has no exchange buffer"
            else:
                try:
                    nat.check(self._lib.marl_dqn_peer_attach(self._h, C.c_int32(rank), C.c_int32(world), b"".join(handles)), "marl_dqn_peer_attach")
                except nat.NativeError as e:
                    err = str(e)
        errors = [None] * world
        dist.all_gather_object(errors, err, group=group)   # agree on the outcome: one collective, reached by every rank
        failed = [f"rank {r}: {e}" for r, e in enumerate(errors) if e is not None]
        if failed:
            raise nat.NativeError("peer-memory gradient exchange unavailable: " + "; ".join(failed))
        self.peers_attached = True
        dist.barrier(group)

    def peer_timed_out(self) -> bool:
        """True when an in-kernel gradient exchange gave up waiting for a peer (bounded spin): every result since is invalid."""
        v = C.c_int32()
        nat.check(self._lib.marl_dqn_peer_status(self._h, C.byref(v)), "marl_dqn_peer_status")
        return bool(v.value)

    def timing_kernels(self):
        """After timing(False): (ms of online forward + TD head, ms of dH1 + dW1, ms of the other weight gradients), launches -- tensor-core pass only."""
        ms3, n = (C.c_float * 3)(), C.c_int32()
        nat.check(self._lib.marl_dqn_timing_kernels(self._h, ms3, C.byref(n)), "marl_dqn_timing_kernels")
        return [float(x) for x in ms3], int(n.value)

    @property
    def updates(self) -> int:
        u = C.c_int64()
        nat.check(self._lib.marl_dqn_counters(self._h, C.byref(u), None), "marl_dqn_counters")
        return int(u.value)

    def hard_update(self):
        nat.check(self._lib.marl_dqn_sync_target(self._h, nat.stream_ptr()), "marl_dqn_sync_target")

    def params_changed(self):
        """Call after writing `theta` / `theta_tgt` directly (checkpoint load, tests): cached derived data is rebuilt."""
        nat.check(self._lib.marl_dqn_params_changed(self._h), "marl_dqn_params_changed")

    def state_dict(self):
        sd = flat_to_state_dict(self.theta.detach().cpu(), f"critic.{self._kind}", self.n_nets, self._shapes)
        sd.update(flat_to_state_dict(self.theta_tgt.detach().cpu(), f"target.{self._kind}", self.n_nets, self._shapes))
        return sd

    def load_state_dict(self, sd):
        for dst, prefix in ((self.theta, "critic"), (self.theta_tgt, "target")):
            dst.copy_(state_dict_to_flat(sd, f"{prefix}.{self._kind}", self.n_nets, self._shapes))
        self.params_changed()


class VDNetwork(QNetwork):
    """marlbase/dqn/model.py:199-269: Q_tot = sum_i Q_i, reward of agent 0 (CooperativeReward makes them equal)."""

    mixer = 1


MIXER_KEYS = ("hyper_w_1.0", "hyper_w_1.2", "hyper_w_final.0", "hyper_w_final.2", "hyper_b_1", "V.0", "V.2")
MIXER_KEYS_1 = ("hyper_w_1", "hyper_w_final", "hyper_b_1", "V.0", "V.2")   # hypernet_layers == 1


def mixer_keys(hypernet_layers=2):
    return MIXER_KEYS if hypernet_layers == 2 else MIXER_KEYS_1


def mixer_shapes(n_agents, state_dim, embed_dim, hypernet_embed, hypernet_layers=2):
    """(out, in) of the mixing network's Linear layers in the reference's state_dict order (dqn/model.py:283-311): seven with two-layer
    hypernetworks, five with one (hyper_w_1 = Linear(S, N*E), hyper_w_final = Linear(S, E); hypernet_embed unused)."""
    N, S, E, He = n_agents, state_dim, embed_dim, hypernet_embed
    if hypernet_layers == 1:
        return ((N * E, S), (E, S), (E, S), (E, S), (1, E))
    return ((He, S), (N * E, He), (He, S), (E, He), (E, S), (E, S), (1, E))


def check_mixing(obs_space, mixing, standardise_returns):
    """The mixer configurations the QMIX kernels implement (csrc/qmix.cuh): 1..8 agents, a state (the observations side by side) of 1..256
    features, embed_dim and (two-layer hypernetworks) hypernet_embed multiples of 4 up to 64, hypernet_layers 1 or 2.  Anything else fails here,
    in Python, before any native call; marl_dqn_qmix_init checks the same limits and whether the mixer fits shared memory."""
    mixing = dict(mixing)
    N, S = len(obs_space), sum(flatdim(o) for o in obs_space)
    E, hl, He = int(mixing["embed_dim"]), int(mixing["hypernet_layers"]), int(mixing["hypernet_embed"])
    why = []
    if not 1 <= N <= 8:
        why.append("n_agents must be 1..8")
    if not 1 <= S <= 256:
        why.append("state_dim must be 1..256")
    if not (4 <= E <= 64 and E % 4 == 0):
        why.append("embed_dim must be a multiple of 4 up to 64")
    if hl not in (1, 2):
        why.append("hypernet_layers must be 1 or 2")
    elif hl == 2 and not (4 <= He <= 64 and He % 4 == 0):
        why.append("hypernet_embed must be a multiple of 4 up to 64")
    if why:
        raise NotImplementedError(f"QMIX with n_agents={N}, state_dim={S}, embed_dim={E}, hypernet_layers={hl}, hypernet_embed={He}, "
                                  f"standardise_returns={standardise_returns} is not implemented by the mixing kernels: {'; '.join(why)}")


class QMixNetwork(QNetwork):
    """marlbase/dqn/model.py:343-443: the agents' Q-values of the chosen (target: double-Q) actions go through a monotonic mixing network conditioned
    on the state (all observations concatenated); one Adam over critic + mixer, the gradient clip covers the critic only, target updates include
    the mixer.  The mixer runs in qmix.cuh's kernels next to the tensor-core training pass of the agents' networks (csrc/dqn.cu, mixer == 2).
    mixing.hypernet_layers 1 and 2 are the reference's two forms; standardise_returns keeps one statistic per batch entry, as the reference's
    RunningMeanStd(shape=(1,)) does once it has seen a (T, B) batch, so every update must use batch_size == max_batch."""

    mixer = 2

    def __init__(self, obs_space, action_space, cfg, layers, parameter_sharing, use_rnn, use_orthogonal_init, mixing, device, max_batch=None, max_episode_length=None):
        check_mixing(obs_space, mixing, bool(getattr(cfg, "standardise_returns", False)))
        super().__init__(obs_space, action_space, cfg, layers, parameter_sharing, use_rnn, use_orthogonal_init, device, max_batch, max_episode_length)
        mixing = dict(mixing)
        self.embed_dim, self.hypernet_embed = int(mixing["embed_dim"]), int(mixing["hypernet_embed"])
        self.hypernet_layers = int(mixing["hypernet_layers"])
        self.state_dim = self.n_agents * self.in_dim
        with torch.cuda.device(self.device):
            nat.check(self._lib.marl_dqn_qmix_init(self._h, C.c_int32(self.embed_dim), C.c_int32(self.hypernet_layers), C.c_int32(self.hypernet_embed)), "marl_dqn_qmix_init")
        ptrs = [C.c_void_p() for _ in range(5)]
        n = C.c_int64()
        nat.check(self._lib.marl_dqn_qmix_ptrs(self._h, *[C.byref(p) for p in ptrs], C.byref(n)), "marl_dqn_qmix_ptrs")
        self.n_mix = int(n.value)
        self.mix, self.mix_tgt, self.mix_m, self.mix_v = [nat.device_view(p.value, self.n_mix, self.device) for p in ptrs[:4]]
        self.mix_grad = nat.device_view(ptrs[4].value, self.n_mix + 4, self.device)
        # QMixer's layers are plain nn.Linear (PyTorch's default initialisation), created in this order (dqn/model.py:283-311)
        parts = []
        for (o, i) in self._mixer_shapes():
            lin = torch.nn.Linear(i, o)
            parts += [lin.weight.data.reshape(-1), lin.bias.data.reshape(-1)]
        self.mix.copy_(torch.cat(parts).float())
        self.hard_update()

    def optimizer_state(self):
        """QNetwork.optimizer_state() plus the mixer's state under "mixer.<name>" (one optimiser over critic + mixer, as the reference's)."""
        st = super().optimizer_state()
        st.update({f"mixer.{k}": t for k, t in optimizers.state(self.optimizer_name, self.mix_m, self.mix_v).items()})
        return st

    def _mixer_shapes(self):
        return mixer_shapes(self.n_agents, self.state_dim, self.embed_dim, self.hypernet_embed, self.hypernet_layers)

    def _mixer_sd(self, flat, prefix):
        sd, o = {}, 0
        for k, (no, ni) in zip(mixer_keys(self.hypernet_layers), self._mixer_shapes()):
            sd[f"{prefix}.{k}.weight"] = flat[o:o + no * ni].view(no, ni).clone(); o += no * ni
            sd[f"{prefix}.{k}.bias"] = flat[o:o + no].clone(); o += no
        return sd

    def state_dict(self):
        sd = super().state_dict()
        sd.update(self._mixer_sd(self.mix.detach().cpu(), "mixer"))
        sd.update(self._mixer_sd(self.mix_tgt.detach().cpu(), "target_mixer"))
        return sd

    def load_state_dict(self, sd):
        super().load_state_dict(sd)
        for dst, prefix in ((self.mix, "mixer"), (self.mix_tgt, "target_mixer")):
            dst.copy_(torch.cat([sd[f"{prefix}.{k}.{p}"].reshape(-1).float() for k in mixer_keys(self.hypernet_layers) for p in ("weight", "bias")]))

    def parameters(self):
        return [self.theta, self.mix]

    def exchanged_buffers(self):
        """The agents' buffer and the mixer's [gradient sums | loss numerator | filled count | 2 spare]: the mixer's step divides by its own
        filled count, which the sum makes global."""
        return [self.grad, self.mix_grad]

    def close(self):
        super().close()
        self.mix = self.mix_tgt = self.mix_m = self.mix_v = self.mix_grad = None

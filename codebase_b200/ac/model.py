"""Independent actor-critic learner on the GPU path -- drop-in for marlbase/ac/model.py A2CNetwork (22-246).

Same constructor signature / Hydra `_target_` role (configs/algorithm/ia2c.yaml:8-26) and the reference's
`state_dict()` key names (`actor.independent.{i}.network.…`, `critic.…`, `target_critic.…`; shared: `.networks.{k}.`; recurrent parts:
`actor.independent.{i}.first_layer.weight`, `….rnn.weight_ih_l0`, …).
All arithmetic runs in libmarlb200.so (marl_a2c_*): actor forward, target-critic pass, n-step returns
(utils/utils.py:38-63) or, with `gae_lambda` set, λ-returns, fused forward / loss / backward of critic and actor, Adam, target sync.  No CPU fallback.
`actor.use_rnn` / `critic.use_rnn` make that part the reference's RNNNetwork (one GRU layer), independently of each other.  `actor.layers` and
`critic.layers` are [H, H] with 1 <= H <= 128, each part its own H.
"""
from __future__ import annotations

import ctypes as C
import numbers
import types

import torch

from .. import _native as nat
from .. import optimizers
from ..learner import MAX_AGENTS, NativeLearner, flat_to_state_dict, flatdim, hidden_width, init_flat_params, init_flat_rnn_params, mlp_shapes, rnn_shapes, \
    sharing_to_nets, state_dict_to_flat
from ..native_env import TrajStore


MAX_IN_DIM = 128   # widest actor / critic input of the actor-critic kernels (csrc/learner.cuh kMaxInDim)


def check_input_widths(obs_space, critic):
    """The input widths the actor-critic kernels take: an actor of 1..128 observation features and a critic of 1..128 inputs (a centralised
    critic reads all agents' observations side by side: n_agents x obs).  Anything wider fails here, in Python, before any native call;
    marl_a2c_create checks the same limit."""
    dims = [flatdim(o) for o in obs_space]
    actor_in = max(dims)
    critic_in = sum(dims) if bool(critic.centralised) and len(dims) > 1 else actor_in
    why = []
    if actor_in > MAX_IN_DIM:
        why.append(f"the actor's observation is {actor_in} wide")
    if critic_in > MAX_IN_DIM:
        what = f"the centralised critic's joint observation is {len(dims)} x {actor_in} = {critic_in} wide" if critic_in != actor_in else \
            f"the critic's observation is {critic_in} wide"
        why.append(what)
    if why:
        raise NotImplementedError(f"{'; '.join(why)}: the actor-critic kernels take at most {MAX_IN_DIM} input features")


def gae_lambda(cfg):
    """cfg.gae_lambda: None (absent or null: the reference's n-step returns) or the λ in [0, 1] of the λ-returns that replace them.  Anything else
    raises ValueError here, before any native call."""
    lam = getattr(cfg, "gae_lambda", None)
    if lam is None:
        return None
    if isinstance(lam, bool) or not isinstance(lam, numbers.Real):
        raise ValueError(f"algorithm.gae_lambda must be null or a number in [0, 1], not {lam!r}")
    lam = float(lam)
    if not 0.0 <= lam <= 1.0:
        raise ValueError(f"algorithm.gae_lambda must be in [0, 1], not {lam}")
    return lam


class A2CNetwork(NativeLearner):
    _destroy = "marl_a2c_destroy"

    def __init__(self, obs_space, action_space, cfg, actor, critic, device, max_envs=None, max_episode_length=None):
        self.gae_lambda = gae_lambda(cfg)
        check_input_widths(obs_space, critic)
        self.actor_hidden = hidden_width(actor.layers, "actor.layers", bool(actor.use_rnn))
        self.critic_hidden = hidden_width(critic.layers, "critic.layers", bool(critic.use_rnn))
        self.actor_rnn, self.critic_rnn = bool(actor.use_rnn), bool(critic.use_rnn)
        self._open(obs_space, action_space, cfg, device)
        # critic.centralised (MAA2C / MAPPO, ac/model.py:62-65): every agent's critic reads the concatenation of all agents' observations
        self.centralised = bool(critic.centralised) and self.n_agents > 1
        self.critic_in = self.n_agents * self.in_dim if self.centralised else self.in_dim
        self._actor_shapes = (rnn_shapes if self.actor_rnn else mlp_shapes)(self.in_dim, self.n_actions, self.actor_hidden)
        self._critic_shapes = (rnn_shapes if self.critic_rnn else mlp_shapes)(self.critic_in, 1, self.critic_hidden)
        self.gamma, self.entropy_coef, self.n_steps = float(cfg.gamma), float(cfg.entropy_coef), int(cfg.n_steps)
        self.grad_clip, self.value_loss_coef = cfg.grad_clip, float(cfg.value_loss_coef)
        self.target_update_interval_or_tau = float(cfg.target_update_interval_or_tau)
        self.actor_net = sharing_to_nets(actor.parameter_sharing, self.n_agents)
        self.critic_net = sharing_to_nets(critic.parameter_sharing, self.n_agents)
        self.n_actor_nets, self.n_critic_nets = max(self.actor_net) + 1, max(self.critic_net) + 1
        self._akind = "independent" if not actor.parameter_sharing else "networks"
        self._ckind = "independent" if not critic.parameter_sharing else "networks"
        self.max_envs = int(max_envs or 1024)
        self.max_T = int(max_episode_length or 500)
        acfg = nat.MlpCfg(self.n_agents, self.n_actor_nets, (C.c_int32 * MAX_AGENTS)(*self.actor_net), self.in_dim, self.actor_hidden, self.n_actions)
        ccfg = nat.MlpCfg(self.n_agents, self.n_critic_nets, (C.c_int32 * MAX_AGENTS)(*self.critic_net), self.critic_in, self.critic_hidden, 1)
        hp = nat.A2cHP(float(cfg.lr), self.gamma, float(self.grad_clip or 0.0), self.n_steps, self.entropy_coef, self.value_loss_coef,
                       self.target_update_interval_or_tau, 0.9, 0.999, 1e-8)
        self._h = C.c_void_p()
        with torch.cuda.device(self.device):
            if self.actor_rnn or self.critic_rnn:
                nat.check(self._lib.marl_a2c_create_rnn(C.byref(acfg), C.byref(ccfg), C.byref(hp), C.c_int32(int(self.actor_rnn)), C.c_int32(int(self.critic_rnn)),
                                                        C.c_int32(self.max_envs), C.c_int32(self.max_T), C.c_int32(self.device.index), C.byref(self._h)),
                          "marl_a2c_create_rnn")
            else:
                nat.check(self._lib.marl_a2c_create(C.byref(acfg), C.byref(ccfg), C.byref(hp), C.c_int32(self.max_envs), C.c_int32(self.max_T),
                                                    C.c_int32(self.device.index), C.byref(self._h)), "marl_a2c_create")
        optimizers.apply(self._lib, "marl_a2c_set_optimizer", self._h, self.optimizer_name)
        ptrs = [C.c_void_p() for _ in range(5)]
        na, nc = C.c_int64(), C.c_int64()
        nat.check(self._lib.marl_a2c_param_ptrs(self._h, *[C.byref(p) for p in ptrs], C.byref(na), C.byref(nc)), "marl_a2c_param_ptrs")
        self.n_actor, self.n_critic = int(na.value), int(nc.value)
        n = self.n_actor + self.n_critic
        self.theta = nat.device_view(ptrs[0].value, n, self.device)
        self.theta_tgt = nat.device_view(ptrs[1].value, self.n_critic, self.device)
        self.adam_m, self.adam_v = nat.device_view(ptrs[2].value, n, self.device), nat.device_view(ptrs[3].value, n, self.device)
        self.grad = nat.device_view(ptrs[4].value, n + 4, self.device)
        # each part by its own rule (RNNNetwork: orthogonal on final_layer only), actor first as the reference creates them
        init_a = init_flat_rnn_params if self.actor_rnn else init_flat_params
        init_c = init_flat_rnn_params if self.critic_rnn else init_flat_params
        self.theta[: self.n_actor].copy_(init_a(self.n_actor_nets, self.in_dim, self.n_actions, actor.use_orthogonal_init, self.actor_hidden))
        self.theta[self.n_actor:].copy_(init_c(self.n_critic_nets, self.critic_in, 1, critic.use_orthogonal_init, self.critic_hidden))
        self.soft_update(1.0)
        self._metrics = torch.zeros(6, dtype=torch.float32, device=self.device)
        self.standardise_returns = bool(getattr(cfg, "standardise_returns", False))   # ac/model.py:112-114
        if self.standardise_returns:
            nat.check(self._lib.marl_a2c_standardise_returns(self._h, C.c_int32(1)), "marl_a2c_standardise_returns")
        if self.gae_lambda is not None:
            self.set_gae_lambda(self.gae_lambda)

    def set_gae_lambda(self, lam):
        """λ-returns of `lam` in [0, 1] in place of the n-step returns from the next update on (DESIGN.md §4.4c); None: the n-step returns again"""
        lam = gae_lambda(types.SimpleNamespace(gae_lambda=lam))
        nat.check(self._lib.marl_a2c_set_gae_lambda(self._h, C.c_int32(lam is not None), C.c_float(0.0 if lam is None else lam)), "marl_a2c_set_gae_lambda")
        self.gae_lambda = lam

    def ret_ms(self):
        """(mean[N], var[N], count) of the RunningMeanStd over the returns (standardise_returns), as CPU values."""
        pm, pc = C.c_void_p(), C.c_void_p()
        nat.check(self._lib.marl_a2c_ret_ms_ptrs(self._h, C.byref(pm), C.byref(pc)), "marl_a2c_ret_ms_ptrs")
        ms = nat.device_view(pm.value, 2 * self.n_agents, self.device).cpu()
        cnt = nat.device_view(pc.value, 1, self.device, "<f8").cpu()
        return ms[: self.n_agents], ms[self.n_agents:], float(cnt[0])

    # ---- views into the flat parameter vector ------------------------------------------------------------------
    @property
    def actor_params(self):
        return self.theta[: self.n_actor]

    @property
    def critic_params(self):
        return self.theta[self.n_actor:]

    def scratch(self, n_envs, T):
        """(target values [N,P,T+1], n-step returns [N,P,T], advantages [N,P,T]) of the last update -- device views for tests."""
        ptrs = [C.c_void_p() for _ in range(3)]
        nat.check(self._lib.marl_a2c_scratch_ptrs(self._h, *[C.byref(p) for p in ptrs]), "marl_a2c_scratch_ptrs")
        N = self.n_agents
        return (nat.device_view(ptrs[0].value, N * n_envs * (T + 1), self.device).view(N, n_envs, T + 1),
                nat.device_view(ptrs[1].value, N * n_envs * T, self.device).view(N, n_envs, T),
                nat.device_view(ptrs[2].value, N * n_envs * T, self.device).view(N, n_envs, T))

    # ---- reference API ------------------------------------------------------------------------------------------------
    def init_actor_hiddens(self, batch_size):
        return self._hiddens(self.actor_rnn, batch_size, self.actor_hidden)

    def init_critic_hiddens(self, batch_size, target=False):
        return self._hiddens(self.critic_rnn, batch_size, self.critic_hidden)

    def _forward_rnn(self, which, obs, out, h, h_out):
        if h_out is None:
            width = self.actor_hidden if which == 0 else self.critic_hidden
            h_out = torch.empty(obs.shape[0], self.n_agents, width, dtype=torch.float32, device=self.device)
        nat.check(self._lib.marl_a2c_forward_rnn(self._h, C.c_int32(which), nat.ptr(obs), C.c_int32(obs.shape[0]), nat.ptr(h), nat.ptr(h_out), nat.ptr(out),
                                                 nat.stream_ptr()), "marl_a2c_forward_rnn")
        return out, h_out

    def logits(self, obs: torch.Tensor, out: torch.Tensor | None = None, h: torch.Tensor | None = None, h_out: torch.Tensor | None = None):
        """Actor pass of act (ac/model.py:148-150): obs f32[E,N,D] -> logits f32[E,N,A].
        A recurrent actor takes one step from h f32[E,N,H] (None: the zero state) and returns (logits, h_out); h_out must not be h."""
        E = obs.shape[0]
        if out is None:
            out = torch.empty(E, self.n_agents, self.n_actions, dtype=torch.float32, device=self.device)
        if self.actor_rnn:
            return self._forward_rnn(0, obs, out, h, h_out)
        nat.check(self._lib.marl_a2c_forward_actor(self._h, nat.ptr(obs), C.c_int32(E), nat.ptr(out), nat.stream_ptr()), "marl_a2c_forward_actor")
        return out

    def values(self, obs: torch.Tensor, target: bool = False, h: torch.Tensor | None = None, h_out: torch.Tensor | None = None):
        """get_value (ac/model.py:155-163): obs f32[E,N,D] -> f32[E,N] (centralised critic: each agent's network reads all N x D values of its env).
        A recurrent critic takes one step from h f32[E,N,H] (None: the zero state) and returns (values, h_out)."""
        E = obs.shape[0]
        out = torch.empty(E, self.n_agents, 1, dtype=torch.float32, device=self.device)
        if self.critic_rnn:
            v, h_out = self._forward_rnn(2 if target else 1, obs, out, h, h_out)
            return v.squeeze(-1), h_out
        nat.check(self._lib.marl_a2c_forward_critic(self._h, nat.ptr(obs), C.c_int32(E), C.c_int32(int(target)), nat.ptr(out), nat.stream_ptr()), "marl_a2c_forward_critic")
        return out.squeeze(-1)

    def act(self, inputs, actor_hiddens, action_mask=None):
        """ac/model.py:147-153 for API parity: list of N tensors [P, obs] -> i64[N, P, 1].  The training loop uses the fused
        marl_lbf_rollout_step(policy=2) which samples from the Philox stream inside the env kernel.  A recurrent actor carries actor_hiddens
        (per agent (1, P, H) or None) and returns the new ones."""
        if action_mask is not None:
            raise NotImplementedError("action masks only exist for smaclite in the reference (out of scope)")
        obs = torch.stack([torch.as_tensor(i, dtype=torch.float32, device=self.device) for i in inputs], 1).contiguous()
        if self.actor_rnn:
            logits, h_out = self.logits(obs, h=self._stack_hiddens(actor_hiddens, self.actor_hidden))
            actor_hiddens = self._split_hiddens(h_out)
        else:
            logits = self.logits(obs)
        dist = torch.distributions.Categorical(logits=logits)
        return dist.sample().T.unsqueeze(-1).contiguous(), actor_hiddens

    def update_from_store(self, batch: TrajStore, n_envs: int, step: int):
        """One `model.update(batch, step)` on the device batch (ac/train.py:176)."""
        nat.check(self._lib.marl_a2c_update(self._h, batch.ref(), C.c_int32(n_envs), C.c_int64(int(step)), nat.ptr(self._metrics), nat.stream_ptr()), "marl_a2c_update")
        return self._metrics

    def update_grads(self, batch: TrajStore, n_envs: int):
        nat.check(self._lib.marl_a2c_update_grads(self._h, batch.ref(), C.c_int32(n_envs), nat.stream_ptr()), "marl_a2c_update_grads")

    def update_apply(self, step: int):
        nat.check(self._lib.marl_a2c_update_apply(self._h, C.c_int64(int(step)), nat.ptr(self._metrics), nat.stream_ptr()), "marl_a2c_update_apply")
        return self._metrics

    def update_allreduce(self, batch: TrajStore, n_envs: int, step: int, all_reduce):
        """update_from_store in the two-call form of data-parallel ranks: update_grads, `all_reduce([grad])` (an in-place sum over ranks of the
        gradient sums, loss numerators and filled count), update_apply.  `step` is the global env-step count."""
        self.update_grads(batch, n_envs)
        all_reduce([self.grad])
        return self.update_apply(step)

    def metrics_dict(self, m=None):
        """ac/model.py:241-246 from the device statistics (policy-gradient term, grad norm, entropy, value loss, ...)."""
        m = (self._metrics if m is None else m).tolist()
        actor_loss = m[0] - self.entropy_coef * m[2]
        return {"loss": actor_loss + self.value_loss_coef * m[3], "actor_loss": actor_loss, "value_loss": m[3], "entropy": m[2]}

    def update(self, batch, step):
        """Reference signature (ac/model.py:189): Batch(obss (T+1,P,N*obs), actions (T,P,N), rewards (T,P,N), dones (T+1,P), filled (T,P))."""
        T1, P, ND = batch.obss.shape
        N, D = self.n_agents, self.in_dim
        store = TrajStore(P, N, T1 - 1, D, self.device)
        store.obs.copy_(batch.obss.view(T1, P, N, D).permute(1, 2, 0, 3))
        store.act.copy_(batch.actions.permute(1, 2, 0))
        store.rew.copy_(batch.rewards.permute(1, 2, 0))
        store.done.copy_(batch.dones.permute(1, 0))
        store.filled.copy_(batch.filled.permute(1, 0))
        return self.metrics_dict(self.update_from_store(store, P, step))

    def soft_update(self, t):
        if t != 1.0:
            self.theta_tgt.copy_((1 - t) * self.theta_tgt + t * self.critic_params)
        else:
            nat.check(self._lib.marl_a2c_sync_target(self._h, nat.stream_ptr()), "marl_a2c_sync_target")

    def state_dict(self):
        th, tg = self.theta.detach().cpu(), self.theta_tgt.detach().cpu()
        sd = flat_to_state_dict(th[: self.n_actor], f"actor.{self._akind}", self.n_actor_nets, self._actor_shapes)
        sd.update(flat_to_state_dict(th[self.n_actor:], f"critic.{self._ckind}", self.n_critic_nets, self._critic_shapes))
        sd.update(flat_to_state_dict(tg, f"target_critic.{self._ckind}", self.n_critic_nets, self._critic_shapes))
        return sd

    def load_state_dict(self, sd):
        self.theta[: self.n_actor].copy_(state_dict_to_flat(sd, f"actor.{self._akind}", self.n_actor_nets, self._actor_shapes))
        self.theta[self.n_actor:].copy_(state_dict_to_flat(sd, f"critic.{self._ckind}", self.n_critic_nets, self._critic_shapes))
        self.theta_tgt.copy_(state_dict_to_flat(sd, f"target_critic.{self._ckind}", self.n_critic_nets, self._critic_shapes))


class PPONetwork(A2CNetwork):
    """Independent PPO -- drop-in for marlbase/ac/model.py PPONetwork (249-352; `_target_: ac.model.PPONetwork`, configs/algorithm/ippo.yaml).
    Same networks, rollout and n-step returns as A2CNetwork; `update` re-uses one batch for `num_epochs` optimisation steps with the clipped
    surrogate (marl_ppo_update: collecting-policy log-probabilities once, then per epoch critic pass -> actor pass -> clip + Adam on the device,
    target critic after the last epoch).  Metrics are the epochs' means, as the reference returns them."""

    def __init__(self, obs_space, action_space, cfg, actor, critic, device, max_envs=None, max_episode_length=None):
        super().__init__(obs_space, action_space, cfg, actor, critic, device, max_envs=max_envs, max_episode_length=max_episode_length)
        self.num_epochs, self.ppo_clip = int(cfg.num_epochs), float(cfg.ppo_clip)

    def update_from_store(self, batch: TrajStore, n_envs: int, step: int):
        nat.check(self._lib.marl_ppo_update(self._h, batch.ref(), C.c_int32(n_envs), C.c_int64(int(step)), C.c_int32(self.num_epochs), C.c_float(self.ppo_clip),
                                            nat.ptr(self._metrics), nat.stream_ptr()), "marl_ppo_update")
        return self._metrics

    # marl_ppo_update split per epoch: prepare once, then per epoch epoch_grads(e) -> (exchange) -> epoch_apply(e); with nothing in between the
    # result is update_from_store's, bit for bit
    def prepare(self, batch: TrajStore, n_envs: int):
        """n-step returns and the collecting policy's log-probabilities of the batch (the batch must stay unchanged until the last epoch)."""
        nat.check(self._lib.marl_ppo_prepare(self._h, batch.ref(), C.c_int32(n_envs), nat.stream_ptr()), "marl_ppo_prepare")

    def epoch_grads(self, batch: TrajStore, n_envs: int, epoch: int):
        """Epoch `epoch`'s gradient sums and statistics in `grad`; epoch 0 prepares the batch first."""
        if epoch == 0:
            self.prepare(batch, n_envs)
        nat.check(self._lib.marl_ppo_epoch_grads(self._h, C.c_float(self.ppo_clip), nat.stream_ptr()), "marl_ppo_epoch_grads")

    def epoch_apply(self, step: int, epoch: int):
        """Epoch `epoch`'s optimiser step; the last epoch also updates the target critic and leaves the epochs' mean metrics."""
        nat.check(self._lib.marl_ppo_epoch_apply(self._h, C.c_int64(int(step)), C.c_int32(epoch), C.c_int32(self.num_epochs), nat.ptr(self._metrics),
                                                 nat.stream_ptr()), "marl_ppo_epoch_apply")
        return self._metrics

    def update_grads(self, batch: TrajStore, n_envs: int):
        raise NotImplementedError("PPO takes one optimiser step per epoch: use epoch_grads(batch, n_envs, epoch) / epoch_apply(step, epoch), or update_allreduce")

    def update_apply(self, step: int):
        raise NotImplementedError("PPO takes one optimiser step per epoch: use epoch_grads(batch, n_envs, epoch) / epoch_apply(step, epoch), or update_allreduce")

    def update_allreduce(self, batch: TrajStore, n_envs: int, step: int, all_reduce):
        """update_from_store with one exchange of `grad` per epoch (each epoch is its own optimiser step)."""
        for e in range(self.num_epochs):
            self.epoch_grads(batch, n_envs, e)
            all_reduce([self.grad])
            self.epoch_apply(step, e)
        return self._metrics

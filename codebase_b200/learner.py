"""What the DQN-family learners (dqn.model) and the actor-critic learners (ac.model) share on the host: the network width check, the space and
parameter-sharing helpers, the flat parameter layouts of the reference's FCNetwork and RNNNetwork with their initialisation and `state_dict`
conversion, and `NativeLearner`, the base of the classes that own a native learner handle."""
from __future__ import annotations

import math
import numbers
from collections import OrderedDict

import numpy as np
import torch

from . import _native as nat
from . import optimizers

HIDDEN = 128       # the shipped network's width (layers = [128, 128]) and the widest the kernels take
MAX_AGENTS = nat.MAX_AGENTS   # 32 = MARL_MAX_AGENTS: the most agents (and networks) a learner takes


def hidden_width(layers, what="layers", use_rnn=False) -> int:
    """The hidden width H of `layers` (algorithm.model.layers / actor.layers / critic.layers): the kernels implement two hidden layers of one width
    (an MLP's two Linear layers, or an RNNNetwork's first_layer and GRU, which the reference requires to be equal), 1 <= H <= 128.  Anything else
    fails here, in Python, before any native call; marl_dqn_create / marl_a2c_create check the same range."""
    widths = list(layers)
    ok = len(widths) == 2 and all(isinstance(w, numbers.Integral) and not isinstance(w, bool) for w in widths) and widths[0] == widths[1] and 1 <= widths[0] <= HIDDEN
    if not ok:
        raise NotImplementedError(f"{what}={widths}: the fused kernels implement two hidden layers of one width H, 1 <= H <= {HIDDEN} "
                                  f"(layers = [H, H]; {'first_layer + one H-wide GRU layer' if use_rnn else 'MLP'})")
    return int(widths[0])


def flatdim(space) -> int:
    """gymnasium.spaces.flatdim for the two space kinds the reference uses (dqn/model.py:32-33)."""
    if getattr(space, "n", None) is not None:
        return int(space.n)
    return int(np.prod(space.shape))


def sharing_to_nets(parameter_sharing, n_agents):
    """utils/models.py:189-196: True -> one network, False -> one per agent, list -> seps indices (renumbered densely)."""
    if parameter_sharing is True:
        return [0] * n_agents
    if parameter_sharing is False or parameter_sharing is None:
        return list(range(n_agents))
    order = []
    for i in parameter_sharing:
        if i not in order:
            order.append(i)
    return [order.index(i) for i in parameter_sharing]


# ---- flat parameter layouts: one network's (state_dict name, shape) in the reference's order; a flat vector holds n_nets of them back to back ----
def mlp_shapes(in_dim, out_dim, hidden=HIDDEN):
    """FCNetwork with layers=[H, H] (utils/models.py:8-48)."""
    H = hidden
    return (("network.0.weight", (H, in_dim)), ("network.0.bias", (H,)), ("network.2.weight", (H, H)), ("network.2.bias", (H,)),
            ("network.4.weight", (out_dim, H)), ("network.4.bias", (out_dim,)))


def rnn_shapes(in_dim, out_dim, hidden=HIDDEN):
    """RNNNetwork with layers=[H, H] (utils/models.py:51-116)."""
    H, H3 = hidden, 3 * hidden
    return (("first_layer.weight", (H, in_dim)), ("first_layer.bias", (H,)), ("rnn.weight_ih_l0", (H3, H)),
            ("rnn.weight_hh_l0", (H3, H)), ("rnn.bias_ih_l0", (H3,)), ("rnn.bias_hh_l0", (H3,)),
            ("final_layer.weight", (out_dim, H)), ("final_layer.bias", (out_dim,)))


def flat_to_state_dict(flat, prefix, n_nets, shapes):
    sd, o = OrderedDict(), 0
    for k in range(n_nets):
        for name, shape in shapes:
            n = int(np.prod(shape))
            sd[f"{prefix}.{k}.{name}"] = flat[o:o + n].view(*shape).clone()
            o += n
    return sd


def state_dict_to_flat(sd, prefix, n_nets, shapes):
    return torch.cat([sd[f"{prefix}.{k}.{name}"].reshape(-1).float() for k in range(n_nets) for name, _ in shapes])


def init_flat_params(n_nets, in_dim, out_dim, use_orthogonal_init=True, hidden=HIDDEN):
    """utils/models.py:8-11,35-44 (host side, once): nn.Linear default init, optionally orthogonal(gain sqrt 2) + zero bias."""
    parts = []
    for _ in range(n_nets):
        for o, i in ((hidden, in_dim), (hidden, hidden), (out_dim, hidden)):
            lin = torch.nn.Linear(i, o)
            if use_orthogonal_init:
                torch.nn.init.orthogonal_(lin.weight.data, gain=math.sqrt(2))
                torch.nn.init.constant_(lin.bias.data, 0)
            parts += [lin.weight.data.reshape(-1), lin.bias.data.reshape(-1)]
    return torch.cat(parts).float()


def init_flat_rnn_params(n_nets, in_dim, out_dim, use_orthogonal_init=True, hidden=HIDDEN):
    """RNNNetwork.__init__ (host side, once): first_layer and the GRU keep PyTorch's default initialisation; use_orthogonal_init applies to
    final_layer only (orthogonal, gain sqrt 2, zero bias).  Modules are created in the reference's order, so the RNG stream matches."""
    parts = []
    for _ in range(n_nets):
        first, gru, final = torch.nn.Linear(in_dim, hidden), torch.nn.GRU(hidden, hidden, num_layers=1), torch.nn.Linear(hidden, out_dim)
        if use_orthogonal_init:
            torch.nn.init.orthogonal_(final.weight.data, gain=math.sqrt(2))
            torch.nn.init.constant_(final.bias.data, 0)
        for t in (first.weight, first.bias, gru.weight_ih_l0, gru.weight_hh_l0, gru.bias_ih_l0, gru.bias_hh_l0, final.weight, final.bias):
            parts.append(t.data.reshape(-1))
    return torch.cat(parts).float()


class NativeLearner:
    """Base of the learners that own a native handle `_h`, destroyed by the C function named `_destroy`.  The subclass creates the handle and
    sets the device views `theta`, `theta_tgt`, `adam_m`, `adam_v` and `grad` of the library-owned buffers."""

    _destroy = None

    def _open(self, obs_space, action_space, cfg, device):
        """The constructors' shared prologue: optimiser name, device (the GPU learners have no CPU fallback), agents and their space sizes.
        More than MAX_AGENTS agents fail here, before any native call (marl_dqn_create / marl_a2c_create refuse them too)."""
        self.n_agents = len(obs_space)
        if self.n_agents > MAX_AGENTS:
            raise NotImplementedError(f"{self.n_agents} agents: the learners take at most {MAX_AGENTS} agents (MARL_MAX_AGENTS)")
        self.optimizer_name = optimizers.optimizer_name(getattr(cfg, "optimizer", "Adam"))
        if not torch.cuda.is_available() or not str(device).startswith("cuda"):
            raise nat.NativeError("the GPU learners need algorithm.model.device=cuda (no CPU fallback)")
        self.device = torch.device(device if ":" in str(device) else f"cuda:{torch.cuda.current_device()}")
        obs_dims, act_dims = [flatdim(o) for o in obs_space], [flatdim(a) for a in action_space]
        if len(set(obs_dims)) != 1 or len(set(act_dims)) != 1:
            raise NotImplementedError("agents with different observation / action sizes are not implemented")
        self.in_dim, self.n_actions = obs_dims[0], act_dims[0]
        self._lib = nat.lib()

    def optimizer_state(self):
        """The optimiser state by torch's names (Adam / AdamW: exp_avg, exp_avg_sq; RMSprop: square_avg; Adagrad: sum; SGD: none), flat
        [n_params] device views in the layout of `theta`."""
        return optimizers.state(self.optimizer_name, self.adam_m, self.adam_v)

    def _hiddens(self, recurrent, batch_size, width):
        """utils/models.py:98-103: zeros (num_layers=1, batch, H) per agent for a recurrent network, None per agent otherwise."""
        if not recurrent:
            return [None] * self.n_agents
        return [torch.zeros(1, batch_size, width, dtype=torch.float32, device=self.device) for _ in range(self.n_agents)]

    def _stack_hiddens(self, hiddens, width):
        """act's hidden states, per agent (1, E, H) or None, as one f32[E, N, H] (None: the zero state)."""
        if hiddens is None or all(x is None for x in hiddens):
            return None
        return torch.stack([torch.as_tensor(x, device=self.device).reshape(-1, width) for x in hiddens], 1).float().contiguous()

    def _split_hiddens(self, h):
        """f32[E, N, H] -> per agent (1, E, H)."""
        return [h[:, i].unsqueeze(0).clone() for i in range(self.n_agents)]

    def parameters(self):
        return [self.theta]

    def close(self):
        if getattr(self, "_h", None):
            getattr(self._lib, self._destroy)(self._h)
            self._h = None
            # the views aliased library-owned device memory that no longer exists
            self.theta = self.theta_tgt = self.adam_m = self.adam_v = self.grad = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

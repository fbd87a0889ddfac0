"""`algorithm.optimizer` for every learner: the name (or torch.optim class) -> the native optimiser (marl_optimizer, include/marl_b200.h).

The reference builds `torch.optim.<name>(parameters, lr=cfg.lr)` with torch's defaults for everything else (marlbase/dqn/model.py:66-71,
368-371; ac/model.py:103-109).  The learners run the step of five of them on the GPU, with those defaults; any other name fails here, in
Python, before any native call.
"""
from __future__ import annotations

import ctypes as C

from . import _native as nat

# name -> (marl_optimizer.kind, torch's defaults besides lr, torch's state names in adam_m / adam_v order)
_TABLE = {
    "Adam": (0, dict(beta1=0.9, beta2=0.999, eps=1e-8), ("exp_avg", "exp_avg_sq")),
    "AdamW": (1, dict(beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-2), ("exp_avg", "exp_avg_sq")),
    "RMSprop": (2, dict(alpha=0.99, eps=1e-8), (None, "square_avg")),
    "Adagrad": (3, dict(eps=1e-10), (None, "sum")),
    "SGD": (4, dict(), (None, None)),
}
SUPPORTED = tuple(_TABLE)


def optimizer_name(opt) -> str:
    """cfg.optimizer as the reference reads it: a torch.optim class name or the class itself.  Raises NotImplementedError for any optimiser
    the learners do not implement."""
    name = opt if isinstance(opt, str) else getattr(opt, "__name__", repr(opt))
    if name not in _TABLE:
        raise NotImplementedError(f"optimizer={name!r} is not implemented; the GPU learners implement {', '.join(SUPPORTED)} "
                                  f"(torch.optim defaults, lr=algorithm.lr)")
    return name


def native(name: str) -> nat.Optimizer:
    kind, consts, _ = _TABLE[name]
    return nat.Optimizer(kind, consts.get("beta1", 0.0), consts.get("beta2", 0.0), consts.get("alpha", 0.0), consts.get("eps", 0.0),
                         consts.get("weight_decay", 0.0))


def apply(lib, setter: str, handle, name: str):
    """marl_dqn_set_optimizer / marl_a2c_set_optimizer right after the handle's creation"""
    o = native(name)
    nat.check(getattr(lib, setter)(handle, C.byref(o)), setter)


def state(name: str, m, v) -> dict:
    """the optimiser state as torch names it (device views of m / v; SGD has none)"""
    return {k: t for k, t in zip(_TABLE[name][2], (m, v)) if k is not None}

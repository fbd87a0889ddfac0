"""Oracle of the optimisers besides Adam (algorithm.optimizer): torch.optim's single-tensor steps with torch's defaults, restated over flat
parameter vectors next to oracle.learner_ref.adam_step, and the oracle learners run with any of them.  TEST INFRASTRUCTURE ONLY.

Each step has adam_step's signature (theta, m, v, grad, step, lr): the state torch keeps goes where the device keeps it -- RMSprop's square_avg
and Adagrad's sum in v; SGD keeps none.  `optimizer(name)` makes learner_ref's and qmix_ref's updates (dqn_update, a2c_update, ppo_update,
qmix_update) take that step instead of Adam's, for both their parts (actor and critic; agents' networks and mixer)."""
from __future__ import annotations

import contextlib

from oracle import learner_ref as lr
from oracle import qmix_ref as qr


def adamw_step(theta, m, v, grad, step, lr_, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=1e-2):
    """torch.optim.AdamW = Adam with decoupled weight decay: param.mul_(1 - lr * weight_decay), then the Adam step"""
    theta.mul_(1 - lr_ * weight_decay)
    _ADAM(theta, m, v, grad, step, lr_, beta1, beta2, eps)


def rmsprop_step(theta, m, v, grad, step, lr_, alpha=0.99, eps=1e-8):
    """torch.optim.RMSprop (centered False, momentum 0): square_avg in v"""
    v.mul_(alpha).addcmul_(grad, grad, value=1 - alpha)
    avg = v.sqrt().add_(eps)
    theta.addcdiv_(grad, avg, value=-lr_)


def adagrad_step(theta, m, v, grad, step, lr_, eps=1e-10, lr_decay=0.0):
    """torch.optim.Adagrad (initial_accumulator_value 0): sum in v"""
    clr = lr_ / (1 + (step - 1) * lr_decay)
    v.addcmul_(grad, grad, value=1)
    std = v.sqrt().add_(eps)
    theta.addcdiv_(grad, std, value=-clr)


def sgd_step(theta, m, v, grad, step, lr_):
    """torch.optim.SGD (momentum 0): no state"""
    theta.add_(grad, alpha=-lr_)


_ADAM = lr.adam_step
STEPS = {"Adam": _ADAM, "AdamW": adamw_step, "RMSprop": rmsprop_step, "Adagrad": adagrad_step, "SGD": sgd_step}
NAMES = tuple(STEPS)
# torch's state names, in the order of the device's (m, v) buffers (None: that buffer is unused)
STATE = {"Adam": ("exp_avg", "exp_avg_sq"), "AdamW": ("exp_avg", "exp_avg_sq"), "RMSprop": (None, "square_avg"), "Adagrad": (None, "sum"),
         "SGD": (None, None)}


@contextlib.contextmanager
def optimizer(name="Adam"):
    """run learner_ref / qmix_ref (and the oracles built on them) with optimiser `name`"""
    saved = lr.adam_step
    lr.adam_step = STEPS[name]
    try:
        yield
    finally:
        lr.adam_step = saved


def dqn_update(st, batch, hp, optimizer_name="Adam"):
    with optimizer(optimizer_name):
        return lr.dqn_update(st, batch, hp)


def qmix_update(st, batch, hp, optimizer_name="Adam"):
    with optimizer(optimizer_name):
        return qr.qmix_update(st, batch, hp)


def a2c_update(st, batch, hp, step, optimizer_name="Adam"):
    with optimizer(optimizer_name):
        return lr.a2c_update(st, batch, hp, step)


def ppo_update(st, batch, hp, step, num_epochs=4, ppo_clip=0.2, optimizer_name="Adam"):
    with optimizer(optimizer_name):
        return lr.ppo_update(st, batch, hp, step, num_epochs, ppo_clip)

"""λ-returns (algorithm.gae_lambda) restated for the tests.  TEST INFRASTRUCTURE ONLY.

The reference has no λ-return; the project defines it (DESIGN.md §4.4c) as the mixture of the reference's own n-step returns
(utils/utils.py:38-63 compute_nstep_returns, oracle/learner_ref.nstep_returns):

    R_t = (1 - λ) Σ_{n>=1} λ^(n-1) G_t^(n)

with m_t = 1 - dones[t] masking reward t and value t, and no term at an index >= T.  For n >= T - t every G_t^(n) is the return to the end of the
stored episode, so the infinite sum is (1 - λ) Σ_{n=1}^{T-1} λ^(n-1) G^(n) + λ^(T-1) G^(T).  `lambda_returns` evaluates exactly that, every
G^(n) from its definition, in float64, streamed over n (O(T x sequences) memory, O(T² x sequences) time): it shares no arithmetic with the
kernel's backward recursion.

`lambda_returns_in(lam)` runs oracle.learner_ref's A2C / PPO updates with these returns in place of the n-step returns (their other arithmetic
unchanged: the de-standardised target values, the running statistics, the losses); it composes with tests/gru_ac_ref.mixed().
"""
from __future__ import annotations

import contextlib

import numpy as np
import torch

from oracle import learner_ref as lr


def nstep_each(rewards, done, next_values, gamma):
    """G^(n) for n = 1 .. T in turn, float64: rewards (T, ...), done and next_values (>= T, ...) -> yields (n, G^(n)) with G^(n) of shape (T, ...).
    G_t^(n) = Σ_{k<n, t+k<T} γ^k m_{t+k} r_{t+k} + [t+n < T] γ^n m_{t+n} V_{t+n}: compute_nstep_returns term by term, vectorised over t.  Only the
    reward sum is kept from one n to the next, so memory is O(T x sequences)."""
    r = np.asarray(rewards, np.float64)
    T = r.shape[0]
    m = 1.0 - np.asarray(done, np.float64)[:T]
    mr, mv = m * r, m * np.asarray(next_values, np.float64)[:T]

    def shifted(x, k):   # x[t + k], zero at t + k >= T
        out = np.zeros_like(x)
        if k < T:
            out[: T - k] = x[k:]
        return out

    rewards_part = np.zeros_like(r)
    for n in range(1, T + 1):
        rewards_part = rewards_part + gamma ** (n - 1) * shifted(mr, n - 1)
        yield n, rewards_part + gamma ** n * shifted(mv, n)


def nstep_all(rewards, done, next_values, gamma):
    """every G^(n) of nstep_each at once: (T, T, ...) with [n - 1] = G^(n) (small T only)"""
    return np.stack([G for _, G in nstep_each(rewards, done, next_values, gamma)])


def lambda_returns(rewards, done, next_values, lam, gamma):
    """(1 - λ) Σ_{n=1}^{T-1} λ^(n-1) G^(n) + λ^(T-1) G^(T), float64 (T, ...), accumulated over n without keeping the G^(n)"""
    T = np.asarray(rewards).shape[0]
    out = 0.0
    for n, G in nstep_each(rewards, done, next_values, gamma):
        out = out + (lam ** (T - 1) if n == T else (1.0 - lam) * lam ** (n - 1)) * G
    return out


def recursion(rewards, done, next_values, lam, gamma):
    """the backward recursion R_t = m_t r_t + γ((1 - λ) m_{t+1} V_{t+1} + λ R_{t+1}), R_T = 0, m_T V_T = 0, float64 -- written out by hand"""
    r = np.asarray(rewards, np.float64)
    d, v = np.asarray(done, np.float64), np.asarray(next_values, np.float64)
    T = r.shape[0]
    out = np.zeros_like(r)
    nxt = np.zeros_like(r[0])
    for t in reversed(range(T)):
        boot = (1.0 - d[t + 1]) * v[t + 1] if t + 1 < T else 0.0
        nxt = (1.0 - d[t]) * r[t] + gamma * ((1.0 - lam) * boot + lam * nxt)
        out[t] = nxt
    return out


@contextlib.contextmanager
def lambda_returns_in(lam):
    """learner_ref's updates with the λ-returns of `lam` (None: unchanged, the n-step returns)"""
    if lam is None:
        yield
        return
    saved = lr.nstep_returns

    def returns(rewards, done, next_values, nsteps, gamma):   # nsteps is not used: the λ-returns replace the n-step returns
        return torch.as_tensor(lambda_returns(rewards.numpy(), done.numpy(), next_values.numpy(), lam, gamma), dtype=rewards.dtype)

    lr.nstep_returns = returns
    try:
        yield
    finally:
        lr.nstep_returns = saved


# ---- the goldens: the reference's A2CNetwork / PPONetwork at n_steps = 1 (λ = 0) and n_steps = T (λ = 1) ----------------------------------------
N, D, A, T = 2, 15, 6, 25
# key: (class, seed, batch seed, envs P, env steps of the updates, epochs, grad_clip, parameter sharing, centralised critic, standardise_returns,
#       reference n_steps, the λ it anchors)
GOLDEN_CASES = {
    "a2c_n1": ("A2CNetwork", 21, 31, 10, (0, 2, 3), 1, False, False, False, False, 1, 0.0),
    "a2c_nT_central": ("A2CNetwork", 22, 32, 10, (0, 2, 3), 1, False, False, True, False, T, 1.0),
    "ppo_n1_standardise": ("PPONetwork", 23, 33, 10, (0, 2, 3), 3, False, False, False, True, 1, 0.0),
    "ppo_nT_shared_clip": ("PPONetwork", 24, 34, 12, (0, 2, 5), 4, 0.5, True, False, False, T, 1.0),
}
GOLDEN_METRICS = ("loss", "actor_loss", "value_loss", "entropy")


def golden_state(key):
    """the oracle state a golden case starts from: seeded weights (actor, critic; the target critic a copy of the critic)"""
    from tests.helpers import seeded_params

    _, seed, _, _, _, _, _, sharing, centralised, std, _, _ = GOLDEN_CASES[key]
    n_nets, nets = (1, [0] * N) if sharing else (N, list(range(N)))
    actor, critic = seeded_params(lr, n_nets, D, A, seed), seeded_params(lr, n_nets, N * D if centralised else D, 1, seed + 1)
    return lr.A2CState(actor, critic.clone(), critic.clone(), nets, nets, D, A, centralised=centralised, ret_ms=lr.RunningMeanStdRef((N,)) if std else None)


def golden_batches(key):
    """the device-layout batches of a golden case's updates"""
    from tests.helpers import ac_batch

    _, _, bseed, P, steps, *_ = GOLDEN_CASES[key]
    rng = np.random.default_rng(bseed)
    return [ac_batch(rng, P, N, T, D) for _ in steps]

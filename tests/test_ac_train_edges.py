"""No GPU: the 1e-5 per-block bar of tests/test_ac_train_edges_gpu.py's class sweep can see a single row.

For every class-sweep case, at its shape on 114 and 132 SMs, the float64 oracle's gradient is computed four times: as the device should sum it;
with the last row that carries a loss of one CTA of the case's class (in the actor pass's plan) weighted 0; with the first row of the next CTA of
the same net weighted 2, where that CTA has one; with the first row of a CTA's partial tile -- its row_begin, as train_kernel walks its tiles from the top down -- weighted
0.  A row is weighted by scaling the gradient of its actor's and its critic's outputs on the way back (the forward is unchanged), which is what a
training pass that loses or repeats that row computes.  Each of the three must miss the bar in at least one block: the rows carry a loss (the
edge episodes run their full length, and row t = 0 of every episode is filled) and are large enough to be seen among up to 20 000 rows."""
import contextlib
import copy
import types

import numpy as np
import pytest
import torch

from codebase_b200.learner import mlp_shapes
from oracle import learner_ref as lr
from tests import gru_ac_ref as gar
from tests import row_plan as rp
from tests import test_ac_train_edges_gpu as ae
from tests import test_agent_range_gpu as ar
from tests import test_rnn_ac_gpu as rac

SEED = 0xAC_ED6E


@contextlib.contextmanager
def _weighted(weights):
    """learner_ref's networks with the gradient of row (agent, b, t) of every differentiated pass (the actor's logits, the critic's values)
    scaled by weights[(agent, b, t)]"""
    def forward(flat, agent_net, xs, in_dim, out_dim):
        out = gar.agents_forward(flat, agent_net, xs, in_dim, out_dim)
        if not flat.requires_grad or not weights:
            return out
        res = []
        for a, y in enumerate(out):
            w = torch.ones(y.shape[0], y.shape[1], 1, dtype=y.dtype)
            for (agent, b, t), v in weights.items():
                if agent == a:
                    w[t, b, 0] = v
            res.append(y * w + y.detach() * (1 - w))
        return res

    saved = lr.agents_forward
    lr.agents_forward = forward
    try:
        yield
    finally:
        lr.agents_forward = saved


def _setup(c, P, T, sm):
    """(the raw gradient of the case's first update at (P, T) on sm SMs, from seeded perturbed parameters with the target critic apart from the
    critic: a function, each call from the same state; the blocks it is judged by; the oracle's batch)"""
    torch.manual_seed(SEED + P + T)
    s, _ = ae.data(c, P, T, sm, SEED + sm)
    b64 = ae._batch64(s, P)
    an, cn = rp.nets_of(c.N, c.sharing), rp.nets_of(c.N, c.csharing)
    actor, critic = lr.init_flat(max(an) + 1, c.D, c.A).double(), lr.init_flat(max(cn) + 1, c.joint, 1).double()
    target = critic + 0.01 * torch.randn_like(critic)
    actor, critic = actor + 0.01 * torch.randn_like(actor), critic + 0.01 * torch.randn_like(critic)   # as ae.perturb: no zero bias
    st = lr.A2CState(actor, critic, target, an, cn, c.D, c.A, centralised=c.kind in ae.CENTRAL,
                     ret_ms=ar._ret_ms64((c.N,)) if c.standardise else None)
    hp = rac._hp(ar._rcase(ae.acase(c, P, T)))

    def grad():
        if c.kind in ae.PPO:
            g = lr.ppo_update(copy.deepcopy(st), b64, hp, 0, 1, 0.2)["grads"][0]
        else:
            g = lr.a2c_update(copy.deepcopy(st), b64, hp, 0)["grad"]
        return np.concatenate([g["actor"].numpy(), g["critic"].numpy()])

    m = types.SimpleNamespace(n_actor_nets=max(an) + 1, n_critic_nets=max(cn) + 1, _actor_shapes=mlp_shapes(c.D, c.A), _critic_shapes=mlp_shapes(c.joint, 1))
    blocks = [(name, sl) for name, sl in ar._blocks(m) if not name.startswith("critic") or not name.endswith(m._critic_shapes[-1][0])]
    return grad, blocks, b64   # (the critic's one-element output bias is judged on a floor on the device: _critic_bias_floors)


def _moved(grad_fn, weights, blocks, want):
    """the largest block move of the weighted gradient against `want`, in bars"""
    with _weighted(weights):
        got = grad_fn()
    return max(float(np.abs(got[sl] - want[sl]).max()) / (ar.BLOCK_TOL * max(float(np.abs(want[sl]).max()), 1e-30)) for _, sl in blocks)


def _row(p, net, r, P, T):
    """row r of net -> (agent, b, t): units are agent-major, unit u of a net is episode u % P of its (u // P)-th agent"""
    unit = r // (T + 1)
    return p["slot_agent"][p["slot_begin"][net] + unit // P], unit % P, r % (T + 1)


def _edge_rows(c, P, T, sm):
    """(what, row, weight) of the three perturbations of the case in the actor pass's plan on sm SMs"""
    p = rp.episode_plan(rp.nets_of(c.N, c.sharing), P, T, sm)
    rows = [(i, net, r0, r1) for i, (net, r0, r1) in enumerate(rp.all_cta_rows(p)) if r1 > r0]
    of_cls = [x for x in rows if c.cls not in rp.CLASSES or (rp.tail_counts(x[3] - x[2]) and rp.classes(x[3] - x[2]) == c.cls)]
    assert of_cls, (c.cls, sm)
    nxt = {i: (net, r0) for i, net, r0, _ in rows}
    i, net, r0, r1 = next((x for x in of_cls if x[0] + 1 in nxt and nxt[x[0] + 1][0] == x[1]), of_cls[0])
    last = r1 - 1 - next(k for k in range(T + 1) if (r1 - 1 - k) % (T + 1) < T)
    out = [(f"the last loss row of CTA {i} ({r0}..{r1 - 1})", _row(p, net, last, P, T), 0.0)]
    if i + 1 in nxt and nxt[i + 1][0] == net:
        out.append((f"the first row of CTA {i + 1}", _row(p, net, nxt[i + 1][1], P, T), 2.0))
    j, jnet, j0, _ = next((x for x in of_cls + rows if (x[3] - x[2]) % rp.TILE), of_cls[0])
    out.append((f"row_begin of CTA {j}", _row(p, jnet, j0, P, T), 0.0))
    return out


@pytest.mark.parametrize("n_sm", [114, 132])
@pytest.mark.parametrize("cls", list(ae.CLASS_CASES))
def test_one_row_misses_the_bar(cls, n_sm):
    c = ae.dataclasses.replace(ae.CLASS_CASES[cls], cls=cls)
    P, T = rp.find_batch(c.N, c.sharing, c.T_choices, n_sm, cls, ae.MAX_ROWS)
    edges = _edge_rows(c, P, T, n_sm)
    grad_fn, blocks, b64 = _setup(c, P, T, n_sm)
    want = grad_fn()
    moves = []
    for what, (agent, b, t), w in edges:
        assert t < T and b64["filled"][t, b] == 1, (cls, n_sm, what, agent, b, t)   # the row carries a loss
        moved = _moved(grad_fn, {(agent, b, t): w}, blocks, want)
        moves.append(f"{what} (agent {agent}, b {b}, t {t}) x {w:g}: {moved:.1f}")
        assert moved > 1.0, f"{cls} on {n_sm} SMs (P={P}, T={T}): {what} weighted {w:g} moves no block past the bar ({moved:.2f})"
    print(f"{cls} on {n_sm} SMs (P={P}, T={T}), worst block moves in bars: " + "; ".join(moves))

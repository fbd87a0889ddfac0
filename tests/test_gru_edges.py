"""No GPU: the 1e-5 per-block bar of tests/test_gru_edges_gpu.py's class sweep can see a single sequence.

For every class-sweep case, at its shape on 114 and 132 SMs, the float64 oracle's gradient is computed three times: as the device should sum it,
without the last sequence of one CTA (of the case's class where there is one, followed by another CTA of its net where there is one), and with the first sequence of the next CTA of the same net
counted twice.  A sequence is left out or doubled by weighting its outputs' gradient 0 or 2 on the way back (the forward is unchanged), which is
what a backward that loses or repeats that sequence computes.  Each of the two must miss the bar in at least one block: the edge sequences carry
gradient (their episodes are filled at every step) and are large enough to be seen among up to ~6000 sequences."""
import contextlib
import copy
import types

import numpy as np
import pytest
import torch

from codebase_b200.learner import mlp_shapes, rnn_shapes
from oracle import learner_ref as lr
from oracle import qmix_ref as qr
from tests import gru_ac_ref as gar
from tests import row_plan as rp
from tests import test_agent_range_gpu as ar
from tests import test_gru_edges_gpu as ge
from tests import test_rnn_ac_gpu as rac
from tests.helpers import ac_oracle_batch

SEED = 0x6A0_ED6E


@contextlib.contextmanager
def _weighted(part, weights):
    """learner_ref's networks (tests/gru_ac_ref.py, any kind and width) with the gradient of sequence (agent, b) of the networks of `part`
    ((in_dim, out_dim)) scaled by weights[(agent, b)]"""
    def forward(flat, agent_net, xs, in_dim, out_dim):
        out = gar.agents_forward(flat, agent_net, xs, in_dim, out_dim)
        if (in_dim, out_dim) != part or not flat.requires_grad:
            return out
        res = []
        for a, y in enumerate(out):
            w = torch.ones(1, y.shape[1], 1, dtype=y.dtype)
            for (agent, b), v in weights.items():
                if agent == a:
                    w[0, b, 0] = v
            res.append(y * w + y.detach() * (1 - w))
        return res

    saved = lr.agents_forward
    lr.agents_forward = forward
    try:
        yield
    finally:
        lr.agents_forward = saved


def _setup(c, B, sm):
    """(the raw gradient of the case's first update at B on sm SMs, from seeded parameters with online != target: a function, each call from the
    same state; the blocks it is judged by)"""
    torch.manual_seed(SEED + B)
    nets = rp.nets_of(c.N, c.sharing)
    n_nets = max(nets) + 1
    s, _ = ge.data(c, B, sm, SEED + sm)
    ac = ge.acase(c, B)
    if c.dqn:
        theta = gar.init_part(True, n_nets, c.D, c.A).double()
        tgt = theta + 0.01 * torch.randn_like(theta)
        b64 = ar._f64(lr.batch_from_store(s, np.arange(B)))
        hp = ge.dqn_hp(c)
        blocks = ar._blocks(types.SimpleNamespace(n_nets=n_nets, _shapes=rnn_shapes(c.D, c.A, c.H)))
        if c.kind == "qmix":
            mix = qr.init_mixer_flat(c.N, c.N * c.D, ge.rdq.MIXING["embed_dim"], ge.rdq.MIXING["hypernet_embed"]).double()
            st = ge.qmix_state(c, theta, tgt, mix, mix + 0.01 * torch.randn_like(mix))
            return (lambda: qr.qmix_update(copy.deepcopy(st), b64, hp)["grad"].numpy()), blocks
        st = lr.DqnState(theta, tgt, nets, c.D, c.A)
        return (lambda: lr.dqn_update(copy.deepcopy(st), b64, hp)["grad"].numpy()), blocks
    CD = c.N * c.D if c.kind in ge.CENTRAL and c.N > 1 else c.D
    actor = gar.init_part(c.arnn, n_nets, c.D, c.A).double()
    critic = gar.init_part(c.crnn, n_nets, CD, 1).double()
    st = lr.A2CState(actor, critic, critic + 0.01 * torch.randn_like(critic), nets, nets, c.D, c.A, centralised=c.kind in ge.CENTRAL)
    b64 = ar._f64(ac_oracle_batch(s))
    hp = rac._hp(ar._rcase(ac))
    m = types.SimpleNamespace(n_actor_nets=n_nets, n_critic_nets=n_nets, _actor_shapes=(rnn_shapes if c.arnn else mlp_shapes)(c.D, c.A, c.H),
                              _critic_shapes=(rnn_shapes if c.crnn else mlp_shapes)(CD, 1, c.critic_H))

    def grad():
        if c.kind in ge.PPO:
            g = lr.ppo_update(copy.deepcopy(st), b64, hp, 0, 1, 0.2)["grads"][0]
        else:
            g = lr.a2c_update(copy.deepcopy(st), b64, hp, 0)["grad"]
        return np.concatenate([g["actor"].numpy(), g["critic"].numpy()])

    blocks = [(name, sl) for name, sl in ar._blocks(m) if not name.startswith("critic") or not name.endswith(m._critic_shapes[-1][0])]
    return grad, blocks   # (the critic's one-element output bias is judged on a floor on the device: _critic_bias_floors)


def _moved(grad_fn, part, weights, blocks, want):
    """the largest block move of the weighted gradient against `want`, in bars"""
    with _weighted(part, weights):
        got = grad_fn()
    return max(float(np.abs(got[sl] - want[sl]).max()) / (ar.BLOCK_TOL * max(float(np.abs(want[sl]).max()), 1e-30)) for _, sl in blocks)


@pytest.mark.parametrize("n_sm", [114, 132])
@pytest.mark.parametrize("cls", list(ge.CLASS_CASES))
def test_one_sequence_misses_the_bar(cls, n_sm):
    c = ge.dataclasses.replace(ge.CLASS_CASES[cls], cls=cls)
    B = ge.units(c, n_sm)
    p = rp.gru_plan(rp.nets_of(c.N, c.sharing), B, n_sm)
    rows = rp.all_cta_rows(p)
    of_cls = [i for i, (_, v0, v1) in enumerate(rows) if v1 > v0 and rp.seq_class(v1 - v0) == cls] or [0]
    pick = next((i for i in of_cls if i + 1 < len(rows) and rows[i + 1][0] == rows[i][0]), of_cls[0])   # one with a next CTA of its net
    net, v0, v1 = rows[pick]
    last = rp.seq_of(p, net, v1 - 1)
    nxt = [rp.seq_of(p, n2, w0) for n2, w0, w1 in rows[pick + 1:pick + 2] if n2 == net and w1 > w0]
    edges = rp.cta_edge_sequences(p)
    assert last in edges and all(x in edges for x in nxt)
    grad_fn, blocks = _setup(c, B, n_sm)
    with _weighted(c.part(), {}):
        want = grad_fn()
    what = f"{cls} on {n_sm} SMs (B={B}, CTA {pick} of net {net}: sequences {v0}..{v1 - 1})"
    dropped = _moved(grad_fn, c.part(), {last: 0.0}, blocks, want)
    print(f"{what}: without sequence {last} the worst block moves {dropped:.1f} x the bar", end="")
    assert dropped > 1.0, f"{what}: leaving out sequence {last} moves no block past the bar ({dropped:.2f})"
    if nxt:
        doubled = _moved(grad_fn, c.part(), {nxt[0]: 2.0}, blocks, want)
        print(f"; with sequence {nxt[0]} twice {doubled:.1f} x", end="")
        assert doubled > 1.0, f"{what}: doubling sequence {nxt[0]} moves no block past the bar ({doubled:.2f})"
    print()

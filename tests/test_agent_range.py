"""No GPU: the learners' agent limit on the host and the edges of tests/test_agent_range_gpu.py's shape table.

The C ABI takes 1 to MARL_MAX_AGENTS = 32 agents and networks (marl_mlp_cfg.agent_net has 32 slots).  The Python learners mirror the limit as
codebase_b200.learner.MAX_AGENTS and refuse a 33rd agent with NotImplementedError before any native call (ctypes would otherwise fail to pack
agent_net with an IndexError).  The GPU file's cases are meant to sit on particular edges of the layout arithmetic; this checks they still do."""
import os
import re

import pytest

from oracle import gru_ref as gr
from oracle import learner_ref as lr
from tests import test_agent_range_gpu as g

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FUSED_TAIL = 132 * 512       # parameters the fused reduce + Adam tail covers in one wave on an H100's 132 SMs (kFusedMaxParams = 512 per block)
MAX_OBS_TC = 32              # kMaxObsDim: the tensor-core paths' input tile (and the DQN family's and its GRU kernels' widest input)
MAX_IN = 128                 # kMaxInDim: the actor-critic FP32 kernels' widest input (KP = 128 tiles above 64)
OUT_PAD = 8                  # kOutPad: the widest output head


def _header_max_agents():
    with open(os.path.join(ROOT, "include", "marl_b200.h")) as f:
        return int(re.search(r"^#define MARL_MAX_AGENTS (\d+)", f.read(), re.M).group(1))


def test_max_agents_mirrors_the_header():
    from codebase_b200 import _native as nat
    from codebase_b200 import learner as L

    assert L.MAX_AGENTS == nat.MAX_AGENTS == _header_max_agents() == 32
    assert dict(nat.MlpCfg._fields_)["agent_net"]._length_ == L.MAX_AGENTS


@pytest.mark.parametrize("kind", g.KINDS)
def test_33_agents_raise_not_implemented(kind):
    """before any native call (and before the device check, so this holds without a GPU); 32 agents pass this check"""
    with pytest.raises(NotImplementedError, match=r"33 agents: the learners take at most 32 agents"):
        g._model(g.Case(kind, 33, 3))


def _P(c, critic=False):
    """floats per network: FCNetwork or RNNNetwork with [128, 128] layers"""
    ind, out = (c.joint, 1) if critic else (c.D, c.A)
    return (gr.net_size if c.rnn else lr.net_size)(ind, out)


def test_cases_sit_on_the_edges_they_claim():
    from codebase_b200.learner import sharing_to_nets

    C = g.CASES
    for name, c in C.items():
        assert 1 <= c.N <= 32 and c.B <= 32 and c.T <= 10 and c.A <= OUT_PAD, name
        assert c.D <= (MAX_OBS_TC if c.dqn else MAX_IN) and c.joint <= MAX_IN, name
        assert not c.double_q or c.B * c.T <= 160, f"{name}: double-Q only in a small batch (near-ties grow with the rows)"
    assert [k for k, c in C.items() if c.double_q] == ["idqn_n1_d30"]
    # 32 agents and 32 networks in each learner family, the MLP and the GRU kernels
    for kind in ("idqn", "vdn", "ia2c", "maa2c"):
        assert any(c.kind == kind and c.N == 32 for c in C.values()), kind
    assert C["idqn_rnn_n32"].rnn and C["ia2c_rnn_n32"].rnn and C["vdn_rnn_n8"].rnn
    # the tensor-core backward: D < 32 (column D carries the bias); D = 31 is the widest, with the full kOutPad head; D = 32 runs the FP32 kernel
    assert C["idqn_n16_d31_seps"].tc_backward and C["idqn_n16_d31_seps"].D == MAX_OBS_TC - 1 and C["idqn_n16_d31_seps"].A == OUT_PAD
    assert not C["vdn_n32_d32_shared"].tc_backward and C["vdn_n32_d32_shared"].D == MAX_OBS_TC
    assert all(C[k].tc_backward for k in ("idqn_n1_d30", "idqn_n8_d30", "vdn_n9_d30", "idqn_n32_d3", "idqn_n32_std"))
    # uneven parameter-sharing groups: 13 / 2 / 1 agents
    nets = sharing_to_nets(list(g.SEPS), 16)
    assert sorted(nets.count(k) for k in set(nets)) == [1, 2, 13]
    # the centralised critic's joint input: exactly 128, 126 and 32 (the tensor-core forward's full W1 width); 32 x 5 = 160 is over the limit
    assert C["maa2c_n32_d4"].joint == MAX_IN and C["maa2c_n6_d21"].joint == 126 and C["mappo_n8_d4"].joint == MAX_OBS_TC
    assert g.Case("maa2c", 32, 5).joint == 160 > MAX_IN
    # KP = 128 tiles: an actor input above 64
    assert 64 < C["ia2c_n32_d126"].D <= MAX_IN and 64 < C["ippo_n19_d71"].D <= MAX_IN
    # parameters per network, and the optimiser tail: update_n's cases exceed the fused tail's one wave, N = 1 fits it
    assert _P(C["idqn_n8_d30"]) == 21254 and _P(C["idqn_n32_d3"]) == 17798
    for name, c in g.UPDATE_N.items():
        assert c.N * _P(c) > FUSED_TAIL, name
    assert _P(C["idqn_n1_d30"]) <= FUSED_TAIL
    ia2c = C["ia2c_n32_d126"]
    assert 32 * (_P(ia2c) + _P(ia2c, critic=True)) > FUSED_TAIL
    # standardise_returns at 32 return columns, in both families
    assert C["idqn_n32_std"].standardise and C["ia2c_n32_std"].standardise and C["idqn_n32_std"].N == C["ia2c_n32_std"].N == 32

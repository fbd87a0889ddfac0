"""GPU: the DQN tensor-core training forward computes the target network's outputs, and for QMIX, VDN and standardise_returns the online outputs
the external TD head reads, on the rows it already holds, where separate forward kernels computed them before.  Same instructions on the same
operands: the gradient sums, the loss statistics and the parameters after three updates are bit for bit those of the separate forwards
(tests/golden/make_tc_fused_target.py)."""

import numpy as np
import pytest

from tests.golden.make_tc_fused_target import CASES, OUT, run_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", list(CASES))
def test_fused_target_forward_is_bit_identical(case):
    want = np.load(OUT)
    got = run_case(case)
    assert sorted(got) == sorted(k.split(".", 1)[1] for k in want.files if k.startswith(case + "."))
    for k, v in got.items():
        ref = want[f"{case}.{k}"]
        assert v.shape == ref.shape, (k, v.shape, ref.shape)
        diff = np.flatnonzero(v.view(np.uint32) != ref.view(np.uint32))
        assert diff.size == 0, f"{case}.{k}: {diff.size} values differ, first at {diff[:5]}: {v[diff[:5]]} vs {ref[diff[:5]]}"

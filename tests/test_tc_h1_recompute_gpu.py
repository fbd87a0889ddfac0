"""GPU: the DQN tensor-core training pass rebuilds H1 in its weight-gradient kernel (the forward's own layer-1 wgmma sequence, layer1_tile)
instead of storing it and reading it back.  Same instructions on the same operands: the gradient sums, the loss statistics and the parameters
after three updates are bit for bit those of the pass that stored H1 (tests/golden/make_tc_h1_recompute.py)."""

import numpy as np
import pytest

from tests.golden.make_tc_h1_recompute import CASES, OUT, run_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", list(CASES))
def test_tc_training_pass_is_bit_identical(case):
    want = np.load(OUT)
    got = run_case(case)
    for k, v in got.items():
        ref = want[f"{case}.{k}"]
        assert v.shape == ref.shape, (k, v.shape, ref.shape)
        diff = np.flatnonzero(v.view(np.uint32) != ref.view(np.uint32))
        assert diff.size == 0, f"{case}.{k}: {diff.size} values differ, first at {diff[:5]}: {v[diff[:5]]} vs {ref[diff[:5]]}"
        assert np.array_equal(v, ref)

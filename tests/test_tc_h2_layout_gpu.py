"""GPU: the DQN tensor-core training forward stores H2 in its accumulator-fragment order (one slab of 64-row tiles per CTA, 16-byte stores) and
the weight-gradient kernel stages its chunks from that order, where the forward stored H2 feature-major before.  Only the layout and the moves
change: the gradient sums, the loss statistics and the parameters after three updates are bit for bit those of the feature-major pass, for
IDQN, VDN, QMIX and standardise_returns, one to four networks, one to four layer-1 k-steps, and CTAs of one chunk, of an odd tile count and
with a partial last tile (tests/golden/make_tc_h2_layout.py; the fixture holds a SHA-256 of every array's bytes and a strided sample of its
values)."""

import numpy as np
import pytest

from tests.golden.make_tc_h2_layout import CASES, OUT, SAMPLE_STRIDE, fingerprint, run_case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("case", list(CASES))
def test_h2_fragment_layout_is_bit_identical(case):
    want = np.load(OUT)
    got = run_case(case)
    assert sorted(f"{case}.{k}.sha256" for k in got) == sorted(k for k in want.files if k.startswith(case + ".") and k.endswith(".sha256"))
    for k, v in got.items():
        fp = fingerprint(v)
        ref = {f: want[f"{case}.{k}.{f}"] for f in fp}
        assert int(fp["size"]) == int(ref["size"]), (k, int(fp["size"]), int(ref["size"]))
        diff = np.flatnonzero(fp["sample"].view(np.uint32) != ref["sample"].view(np.uint32))
        assert diff.size == 0, (f"{case}.{k}: {diff.size} sampled values differ, first at {diff[:5] * SAMPLE_STRIDE}: "
                                f"{fp['sample'][diff[:5]]} vs {ref['sample'][diff[:5]]}")
        assert np.array_equal(fp["sha256"], ref["sha256"]), f"{case}.{k}: the sampled values agree, but the array's bytes differ"

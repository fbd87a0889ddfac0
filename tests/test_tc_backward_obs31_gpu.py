"""GPU: the wgmma training pipeline at observation width 31, the widest it takes: the ones line that carries db1 is then the last line of the
[X | 1] operand of the dW1 product.  Same checks as tests/test_tc_backward_gpu.py (gradients, loss and parameters against the fused FP32 kernel
and the CPU oracle), IDQN and VDN, ragged tiles."""
import pytest

from tests import test_tc_backward_gpu as tcb
from tests.test_tc_backward_gpu import _restore  # noqa: F401  (autouse: the library's kernel selection is restored after each case)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("mixer,N,D,T,B,sharing", [(0, 2, 31, 25, 200, False), (1, 3, 31, 25, 96, False)])
def test_tc_backward_obs31_matches_ffma_and_oracle(mixer, N, D, T, B, sharing):
    tcb.test_tc_backward_matches_ffma_and_oracle(mixer, N, D, T, B, sharing)

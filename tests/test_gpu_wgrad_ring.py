"""gemm_tn_kernel's producer / consumer rings held to exact results at the point counts that reach each ring phase.

The split of the points (tn_k_chunk) gives these slice counts per split (32-point slices), with TN_LAND = 4 landing
stages and TN_STAGES = 3 plane stages:
  P = 129:  one split of 5 slices (one more than the landing ring), the last slice holding 1 point;
  P = 513:  splits of 10 and 7 slices (one more than a multiple of the plane stages), a 1-point tail;
  P = 3585: the last split holds a single slice with a single point;
  P = 3617: the last split holds 2 slices (fewer than either ring), the second with 1 point.
Each must reproduce the fp64 sum of the scheme's plane products bit for bit (tests/proto/tc_exact.py), as
test_gpu_tc_exact.py holds the shapes the networks run at."""
import pytest
import torch

from tests.proto import tc_exact as T
from tests.test_gpu_tc_exact import WGRAD_SHAPES, _check_wgrad

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


RING_POINTS = {129: (6, 5), 513: (10, 7), 3585: (16, 1), 3617: (16, 2)}   # P: slices of a whole split, of the last


def _slices(n_out, n_in, P):
    kc = T.tn_k_chunk(n_out, n_in, P)
    last = P - (-(-P // kc) - 1) * kc
    return -(-kc // 32), -(-last // 32)


@pytest.mark.parametrize("n_out,n_in", WGRAD_SHAPES)
@pytest.mark.parametrize("P", sorted(RING_POINTS))
def test_wgrad_exact_ring_phases(P, n_out, n_in):
    assert _slices(n_out, n_in, P) == RING_POINTS[P]
    _check_wgrad(P, n_out, n_in, n_in, "F0", seed=P + n_out + n_in)
    _check_wgrad(P, n_out, n_in, n_in, "F1a", seed=P + n_out + 2)

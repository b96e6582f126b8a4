"""pose_optimize_kernel (csrc/pose_kernels.cu) on the device at every edge case of pose_cases.py, at full size, against
oracle.pose_optimize_trace: the bar of pose_cases.compare (exact for margin-qualified cases, the north-star bar otherwise), the
truth for the noise-free families, and bitwise identical outputs when the same call is repeated (the cluster sums in a fixed order)."""
import pytest

import pose_cases as PC
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S

pytestmark = pytest.mark.gpu
CASES = PC.all_cases()


@pytest.fixture(scope="module")
def ctx():
    c = F.Context(S.KITTI_W, S.KITTI_H, 2000)
    yield c
    c.close()


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_pose_kernel_edges(ctx, c):
    p = c["problem"]
    ref = PC.reference(p)
    PC.check_coverage(c, ref[3])
    got = F.Optimizer.PoseOptimization(ctx, *PC.args(p))
    bar = PC.compare(c, got, ref)
    again = F.Optimizer.PoseOptimization(ctx, *PC.args(p))
    assert again[0] == got[0] and again[1].tobytes() == got[1].tobytes() and again[2].tobytes() == got[2].tobytes()
    print(c["name"], bar)

"""rgbl_local_bundle_adjustment (csrc/api_ba.cu) on the device at every case of ba_cases.py, at full size, against
oracle.local_bundle_adjustment_trace: the bar of ba_cases.compare (exact for margin-qualified cases, 1e-4 otherwise), the truth for the
noise-free cases, and the dense longdouble reference for one LM step.  Every call is repeated on the same context: ba_schur_kernel
accumulates S with atomicAdd on doubles, so the last bits of the FP64 state depend on the order the warps arrive in and the repeat need
not be bitwise equal.  The outputs are float32, so such a difference shows as nothing or as one float32 ulp where a value sits on a
rounding boundary: the repeat must give the same iteration count and flags, and poses and points within one float32 ulp.  Observed on an
H100 (700 W) over two runs of this file: every repeat bitwise equal but one, `far_rotation`, one ulp (2.4e-7) in one translation, once."""
import numpy as np
import pytest

import ba_cases as BC
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S

pytestmark = pytest.mark.gpu
CASES = BC.all_cases()


@pytest.fixture(scope="module")
def ctx():
    c = F.Context(S.KITTI_W, S.KITTI_H, 1000, max_batch=1)
    yield c
    c.close()


def run(ctx, p):
    return F.local_bundle_adjustment(ctx, *BC.args(p)[:-1], iterations=p["iterations"])


def repeat_difference(a, b):
    """Same iterations and flags; -> the largest pose / point difference, in float32 ulps of the value."""
    assert a[3] == b[3] and np.array_equal(a[2], b[2])
    return max(float((np.abs(x.astype(np.float64) - y) / np.spacing(np.maximum(np.abs(x), np.abs(y)))).max()) for x, y in ((a[0], b[0]), (a[1], b[1])))


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_ba_edges(ctx, c):
    p = c["problem"]
    ref = BC.reference(p)
    BC.check_coverage(c, ref[4])
    got = run(ctx, p)
    bar, d_pose, d_pt = BC.compare(c, got, ref)
    BC.truth(c, got[0], got[1])
    dense = BC.compare_dense(c, got[0], got[1]) if c["family"] == "dense" else None
    rep = repeat_difference(got, run(ctx, p))
    assert rep <= 1, (c["name"], rep)
    n_opt = int((p["pose_fixed"] == 0).sum())
    print(f"{c['name']}: cholesky {BC.cholesky_shape(n_opt)} {bar} bar, pose {d_pose:.1e}, point {d_pt:.1e}, repeat {rep:.0f} ulp"
          + (f", dense reference pose {dense[0]:.1e} point {dense[1]:.1e}" if dense else ""))


def test_arena_reuse_across_calls(ctx):
    """Large, small, large again on one context, then a well-posed graph after one whose every factorisation fails: the arena is carved
    anew for every call, so nothing the last call left in it (S, x_p, the status word, the errors) may reach the next result."""
    by_name = {c["name"]: c for c in CASES}
    first = {}
    for name in ("solver64", "solver1", "solver64", "deg_poses", "allzero", "grid_e127", "plane", "solver1", "iters0"):
        c = by_name[name]
        got = run(ctx, c["problem"])
        BC.compare(c, got, BC.reference(c["problem"]))
        if name in first:
            assert repeat_difference(first[name], got) <= 1, name
        first.setdefault(name, got)

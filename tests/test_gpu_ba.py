"""rgbl_local_bundle_adjustment against the oracle: same LM trajectory (iterations), poses / points within 1e-4 relative
(north-star tolerance for floating point), identical erase flags."""
import numpy as np
import pytest

import oracle
import ba_data as D
from orb_slam3_rgbl_b200 import frontend as F, synthetic as S

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = F.Context(S.KITTI_W, S.KITTI_H, 1000, max_batch=1)
    yield c
    c.close()


@pytest.mark.parametrize("seed,n_kf,n_fixed,n_points,out", [(1, 8, 2, 600, 0.03), (2, 12, 3, 1500, 0.05), (3, 4, 1, 80, 0.0), (4, 20, 4, 2500, 0.02),
                                                           (5, 6, 6, 300, 0.03), (6, 3, 1, 12, 0.1)])
def test_matches_oracle(ctx, seed, n_kf, n_fixed, n_points, out):
    p = D.make_problem(seed, n_kf=n_kf, n_fixed=n_fixed, n_points=n_points, outlier_frac=out)
    rpo, rpt, rer, rit, rchi = oracle.local_bundle_adjustment(*D.args(p))
    gpo, gpt, ger, git = F.local_bundle_adjustment(ctx, *D.args(p))
    assert git == rit, (git, rit)
    assert np.abs(gpo - rpo).max() < 1e-4, np.abs(gpo - rpo).max()
    assert np.abs(gpt - rpt).max() < 1e-4 * max(1.0, np.abs(rpt).max()), np.abs(gpt - rpt).max()
    assert np.array_equal(ger, rer), (int((ger != rer).sum()), len(rer))
    assert np.array_equal(gpo[:n_fixed], p["poses"][:n_fixed])


def test_partial_iterations_and_empty_graph(ctx):
    p = D.make_problem(7, n_kf=6, n_points=200)
    for k in (0, 1, 3):
        rpo, rpt, rer, rit, _ = oracle.local_bundle_adjustment(*D.args(p), iterations=k)
        gpo, gpt, ger, git = F.local_bundle_adjustment(ctx, *D.args(p), iterations=k)
        assert git == rit and np.abs(gpo - rpo).max() < 1e-4 and np.abs(gpt - rpt).max() < 1e-3
        assert np.array_equal(ger, rer)
    none = (p["poses"], p["pose_fixed"], p["points"], np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros((0, 3), np.float32),
            np.zeros(0, np.uint8), np.zeros(0, np.float32), *p["cam"])
    gpo, gpt, ger, git = F.local_bundle_adjustment(ctx, *none)
    assert git == 0 and np.array_equal(gpo, p["poses"]) and np.array_equal(gpt, p["points"]) and len(ger) == 0
    bad = list(D.args(p)); bad[3] = p["e_point"].copy(); bad[3][0] = len(p["points"])
    with pytest.raises(Exception):
        F.local_bundle_adjustment(ctx, *bad)

"""rgbl_global_bundle_adjustment (csrc/api_ba.cu) and the tiled factorisation (csrc/ba_factor.cu) on the device: every case of gba_cases.py
against the oracle under the bars of gba_cases.compare, each repeated on the same context within one float32 ulp (ba_schur_kernel's
atomicAdd makes the last bits of the FP64 state depend on warp arrival order, see test_gpu_ba_edges.py); local BA above 64 free key frames
(the tiled path) against the local-BA oracle; one LM step against the dense longdouble reference; the solve export against numpy; the
capacity refusal and a call after it."""
import numpy as np
import pytest

import ba_cases as BC
import gba_cases as GC
import gba_dense_reference as GD
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S
from test_gpu_ba_edges import repeat_difference

pytestmark = pytest.mark.gpu
CASES = GC.all_cases()


@pytest.fixture(scope="module")
def ctx():
    c = F.Context(S.KITTI_W, S.KITTI_H, 1000, max_batch=1)
    yield c
    c.close()


def run(ctx, p):
    return F.global_bundle_adjustment(ctx, *GC.args(p), iterations=p["iterations"], robust=p["robust"],
                                      stop=np.array([1 if p["stop"] else 0], np.uint8))


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_gba_cases(ctx, c):
    p = c["problem"]
    ref = GC.reference(p)
    GC.check_coverage(c, ref[3])
    got = run(ctx, p)
    bar, d_pose, d_pt = GC.compare(c, got, ref)
    again = run(ctx, p)
    rep = repeat_difference((got[0], got[1], np.zeros(0), got[2]), (again[0], again[1], np.zeros(0), again[2]))
    assert rep <= 1, (c["name"], rep)
    print(f"{c['name']}: {GC.solver_path(int((p['pose_fixed'] == 0).sum()))} {bar} bar, pose {d_pose:.1e}, point {d_pt:.1e}, repeat {rep:.0f} ulp")


@pytest.mark.parametrize("n_free", [65, 100])
def test_local_ba_on_the_tiled_path(ctx, n_free):
    c = BC.case(f"local{n_free}", "solver", BC.graph(1200 + n_free, 2, n_free, BC.vis_degree(1200 + n_free, 2, n_free, 4 * n_free, 5)), n_opt=n_free)
    ref = BC.reference(c["problem"])
    BC.check_coverage(c, ref[4])
    got = F.local_bundle_adjustment(ctx, *BC.args(c["problem"])[:-1], iterations=c["problem"]["iterations"])
    bar, d_pose, d_pt = BC.compare(c, got, ref)
    print(f"local BA {n_free} free key frames: {bar} bar, pose {d_pose:.1e}, point {d_pt:.1e}")


def test_one_step_matches_the_dense_reference(ctx):
    c = GC.dense_case()
    po, pt, it = run(ctx, c["problem"])
    GC.check_first_accepted(c, GC.reference(c["problem"])[3])
    assert it == 1
    print("dense reference: pose %.1e point %.1e" % GD.compare(c["problem"], po, pt))


def _solve(A, b, path):
    so = L.testing_lib()
    n = len(b); x = np.full(n, np.nan); st = np.full(1, -1, np.int32)
    A = np.ascontiguousarray(A, np.float64); b = np.ascontiguousarray(b, np.float64)
    assert so.rgbl_testing_reduced_solve(n, A.ctypes.data, b.ctypes.data, path, x.ctypes.data, st.ctypes.data) == 0
    return x, int(st[0])


def test_solve_export_against_numpy():
    """n = 1 .. 3 tiles + 5 on the tiled path against numpy; on every n <= 384 both paths agree; a failing pivot in the last tile."""
    rng = np.random.default_rng(7)
    worst = 0.0
    for n in list(range(1, 3 * GC.TILE + 6)) + [250, 320, 383, 384]:
        M = rng.normal(size=(n, n))
        A = M @ M.T + n * np.eye(n)
        b = rng.normal(size=n)
        ref = np.linalg.solve(A, b)
        x2, s2 = _solve(np.tril(A), b, 2)
        x1, s1 = _solve(np.tril(A), b, 1)
        assert s1 == 0 and s2 == 0, n
        e2 = np.abs(x2 - ref).max() / np.abs(ref).max()
        assert e2 < 1e-12 and np.abs(x1 - x2).max() <= 1e-12 * np.abs(ref).max(), (n, e2)
        worst = max(worst, e2)
    for n, bad in ((197, 196), (197, 0), (640, 600)):
        A = np.eye(n)
        A[bad, bad] = 0.0
        x, st = _solve(A, np.ones(n), 2)
        assert st == 1 and not x.any(), (n, bad)
    print(f"tiled solve, worst relative error against numpy {worst:.1e}")


def test_capacity_refusal_then_a_call(ctx):
    p = GC.refused()
    with pytest.raises(L.RgblError) as e:
        run(ctx, p)
    assert e.value.code == L.RGBL_E_CAPACITY
    c = GC.selection()[1]
    GC.compare(c, run(ctx, c["problem"]), GC.reference(c["problem"]))

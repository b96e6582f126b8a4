"""rgbl_local_bundle_adjustment (csrc/api_ba.cu) run through the whole library compiled over the CUDA-on-CPU shim (tests/cuda_emu), so a
machine without a GPU executes its thirteen kernels: a subset of the cases of ba_cases.py against oracle.local_bundle_adjustment_trace
with the bars of ba_cases.compare, one graph against the dense longdouble reference, and, with the oracle alone at full size, that every
case reaches the path it exists for."""
import ctypes as C

import numpy as np
import pytest

import ba_cases as BC
from cuda_emu import build
from orb_slam3_rgbl_b200 import _lib as L


class EmuBA:
    """rgbl_local_bundle_adjustment of the emulated library."""

    def __init__(self, path):
        self.so = C.CDLL(str(path))
        for name, (res, args) in L.SYMBOLS.items():
            fn = getattr(self.so, name)
            fn.restype, fn.argtypes = res, args
        cfg = L.Config(0, 160, 120, 1, 0, 0, L.OrbParams(200, 1.2, 4, 20, 7))
        self.h = C.c_void_p()
        assert self.so.rgbl_create(C.byref(cfg), C.byref(self.h)) == 0

    def __call__(self, poses, fixed, points, e_point, e_pose, obs, stereo, info, fx, fy, cx, cy, bf, iterations):
        po = np.empty_like(poses); pt = np.empty_like(points); er = np.zeros(max(len(e_point), 1), np.uint8); it = C.c_int(0)
        rc = self.so.rgbl_local_bundle_adjustment(self.h, len(poses), L.ptr(poses), L.ptr(fixed), len(points), L.ptr(points), len(e_point), L.ptr(e_point),
                                                  L.ptr(e_pose), L.ptr(obs), L.ptr(stereo), L.ptr(info), fx, fy, cx, cy, bf, iterations, L.ptr(po), L.ptr(pt),
                                                  L.ptr(er), C.byref(it))
        assert rc == 0, self.so.rgbl_last_error(self.h)
        return po, pt, er[:len(e_point)], it.value

    def close(self):
        self.so.rgbl_destroy(self.h)


@pytest.fixture(scope="module")
def emu():
    e = EmuBA(build.build_full())
    yield e
    e.close()


CASES = BC.emulated_cases()


def test_subset_has_every_launch_shape():
    shapes = {BC.cholesky_shape(int((c["problem"]["pose_fixed"] == 0).sum())) for c in CASES}
    assert {("shared", 256), ("global", 256), ("global", 1024)} <= shapes


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_ba_emulated(emu, c):
    p = c["problem"]
    ref = BC.reference(p)
    BC.check_coverage(c, ref[4])
    got = emu(*BC.args(p))
    bar, d_pose, d_pt = BC.compare(c, got, ref)
    BC.truth(c, got[0], got[1])
    print(f"{c['name']}: {bar} bar, pose {d_pose:.1e}, point {d_pt:.1e}")


def test_one_step_matches_the_dense_reference(emu):
    c = next(c for c in BC.dense() if c["name"] == "dense_mixed")
    BC.check_coverage(c, BC.reference(c["problem"])[4])
    po, pt, _, it = emu(*BC.args(c["problem"]))
    assert it == 1
    BC.compare_dense(c, po, pt)


def test_families_reach_their_paths():
    """Through the oracle's trace, at full size: every case reaches what it exists for, the oracle itself takes the dense reference's
    step, and over all cases there is a run of >= 3 rejected trials followed by an accepted one, a qmax == 10 termination, an n_bad stop, a
    rho == 0 stop, failed factorisations, calls ending on a rejected trial with and without qmax == 10, free key-frame counts on both
    sides of 26 / 27 and 32 / 33, and cases on the exact bar in every family that compares poses."""
    traces = {}
    for c in BC.all_cases():
        ref = BC.reference(c["problem"])
        BC.check_coverage(c, ref[4])
        BC.truth(c, ref[0], ref[1])
        if c["family"] == "dense":
            BC.compare_dense(c, ref[0], ref[1])
        traces[c["name"]] = (c, ref[4])
    tr = [t for _, t in traces.values()]
    assert any(t["max_reject_run"] >= 3 and t["trial_accepted"][-1] for t in tr)
    assert any(t["term_qmax"] for t in tr) and any(t["term_nbad"] for t in tr) and any(t["term_rho0"] for t in tr)
    assert any(t["solver_failures"] for t in tr)
    assert any(t["ended_on_rejected_trial"] and t["term_qmax"] for t in tr) and any(t["ended_on_rejected_trial"] and not t["term_qmax"] for t in tr)
    n_opt = {int((c["problem"]["pose_fixed"] == 0).sum()) for c, _ in traces.values()}
    assert {0, 1, 26, 27, 32, 33} <= n_opt and max(n_opt) >= 64
    for fam in ("solver", "degree", "grid", "lm", "numeric", "no_free_pose"):
        assert any(BC.qualifies(t) for c, t in traces.values() if c["family"] == fam), fam

"""pose_optimize_kernel skips the LM rounds that repeat the round before them (no edge level changed, and the same robust flag or no
Huber linear-region evaluation in that round).  Under the CUDA-on-CPU shim the shipped kernel must equal, byte for byte, the same kernel
built with -DPOSE_RUN_ALL_ROUNDS (every round runs): inlier count, float32 pose, outlier flags, edge levels and the errors the last
classification read.  Each case first shows through the per-round trace of the oracle's code (pose_round_trace.py, which runs every round)
that it reaches the path it exists for: rounds skipped after round 0, round 2 skipped alone, round 3 skipped because the linear region was never
reached, and controls that must run their rounds (a level change after round 1, a linear-region hit only at the initial pose, which makes
the skip from round 0 to round 3 start with a build pass of its own, and the n < 10 break)."""
import ctypes as C

import numpy as np
import pytest

import pose_cases as PC
import pose_round_trace as PRT
from cuda_emu import build


def _seeded(seed, outlier_frac):
    """40 edges, small noise, a start close to the truth: few or no edges near Huber's threshold after round 0."""
    return PC.problem(seed, 40, outlier_frac, 0.5, noise=0.2, start_rot=0.01, start_trans=0.1)


# name -> (problem, the trace condition of its path, replica rounds the kernel skips)
PATHS = {
    # no level changes at all and no linear-region evaluation: rounds 1, 2 and 3 repeat round 0
    "clean": (_seeded(6237, 0.0), lambda t: t["changed"] == [0, 0, 0, 0] and t["linear"][0] == 0, 3),
    # nothing changed after round 0, round 0 hit the linear region: rounds 1 and 2 skipped, round 3 runs non-robust; its first system is
    # reused from round 0's classification (no hit at the initial pose) or built anew (hits there)
    "far0": (None, lambda t: t["changed"][0] == 0 and t["linear"][0] > 0, 2),
    "plane1": (None, lambda t: t["changed"][0] == 0 and t["linear"][0] > 0, 2),
    "first_only": (_seeded(6003, 0.0), lambda t: t["changed"][0] == 0 and 0 < t["linear_first"][0] and t["linear"][0] == 2 * t["linear_first"][0]
                   and t["linear_rejected"][0] == 0, 2),
    # a level change after round 0 only: round 2 skipped alone, round 3 runs (round 2 was in the linear region)
    "n10": (None, lambda t: t["changed"][0] > 0 and t["changed"][1] == 0 and t["linear"][2] > 0, 1),
    "n1025": (None, lambda t: t["changed"][0] > 0 and t["changed"][1] == 0 and t["linear"][2] > 0, 1),
    "unconv2": (None, lambda t: t["changed"][0] > 0 and t["changed"][1] == 0 and t["linear"][2] > 0, 1),
    "quat0": (None, lambda t: t["changed"][0] > 0 and t["changed"][1] == 0 and t["linear"][2] > 0, 1),
    # round 1 never reached the linear region and changed nothing: rounds 2 and 3 skipped
    "r23": (_seeded(6726, 0.15), lambda t: t["changed"][0] > 0 and t["changed"][1] == 0 and t["linear"][1] == 0, 2),
    "allout": (None, lambda t: t["changed"][1] == 0 and t["linear"][1] == 0 and t["iters"][1] == 1, 2),
    # controls: a level changed after round 1 (rej0) or after every round (plane0); n = 9 runs one round only
    "rej0": (None, lambda t: t["changed"][1] == 1 and t["changed"][2] == 0 and t["linear"][2] > 0, 0),
    "plane0": (None, lambda t: min(t["changed"][:3]) > 0, 0),
    "n9": (None, lambda t: t["rounds"] == 1, 0),
}
_BY_NAME = {c["name"]: c["problem"] for c in PC.all_cases()}


def _problem(name):
    p = PATHS[name][0]
    return _BY_NAME[name] if p is None else p


class EmuPoseState:
    """emu_pose_optimize of an emulated library: the kernel's outputs and its per-edge state."""

    def __init__(self, path):
        self.so = C.CDLL(str(path))
        self.so.emu_pose_optimize.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 4 + [C.c_float] * 5 + [C.c_void_p] * 5
        self.so.emu_pose_optimize.restype = C.c_int

    def __call__(self, pose, xw, obs, inv_s2, stereo, fx, fy, cx, cy, bf):
        arrs = [np.ascontiguousarray(a, t) for a, t in ((pose, np.float32), (xw, np.float32), (obs, np.float32), (inv_s2, np.float32),
                                                       (stereo, np.uint8))]
        n = len(arrs[1])
        out = np.zeros(7, np.float32); outlier = np.zeros(n, np.uint8); level = np.zeros(n, np.uint8); work = np.zeros(4 * n, np.float64)
        ni = np.zeros(1, np.int32)
        ptr = [a.ctypes.data for a in arrs]
        assert self.so.emu_pose_optimize(ptr[0], n, *ptr[1:], fx, fy, cx, cy, bf, out.ctypes.data, outlier.ctypes.data, level.ctypes.data,
                                         work.ctypes.data, ni.ctypes.data) == 0
        return dict(n_inliers=ni, pose=out, outlier=outlier, level=level, work=work)


@pytest.fixture(scope="module")
def kernels():
    return EmuPoseState(build.build_full()), EmuPoseState(build.build_full(defines=["-DPOSE_RUN_ALL_ROUNDS"]))


@pytest.mark.parametrize("name", list(PATHS))
def test_path_reached(name):
    _, reached, replicas = PATHS[name]
    p = _problem(name)
    *got, t = PRT.pose_optimize_trace(*PC.args(p))
    *want, _ = PC.reference(p)                  # the counters change nothing the oracle computes
    assert got[0] == want[0] and got[1].tobytes() == want[1].tobytes() and got[2].tobytes() == want[2].tobytes(), name
    assert reached(t), (name, t)
    assert t["replica_rounds"] == replicas, (name, t)


@pytest.mark.parametrize("name", list(PATHS))
def test_skipping_equals_every_round(kernels, name):
    a, b = (k(*PC.args(_problem(name))) for k in kernels)          # skipping, every round
    for key in a:
        assert a[key].tobytes() == b[key].tobytes(), (name, key)
    assert (a["level"] == a["outlier"]).all()

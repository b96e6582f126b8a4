"""pose_optimize_kernel (csrc/pose_kernels.cu, PoseOptimization as one thread-block cluster) run through the whole library compiled
over the CUDA-on-CPU shim (tests/cuda_emu): all CTAs of the cluster run at once, the partial sums go through the modelled st.async +
mbarrier exchange.  A subset of the edge cases of pose_cases.py against oracle.pose_optimize_trace, at the shipped cluster shape
(16 CTAs x 64 threads) and at 8 x 128, with the bars of pose_cases.compare; every call is repeated and must give identical outputs."""
import ctypes as C

import numpy as np
import pytest

import pose_cases as PC
from cuda_emu import build
from orb_slam3_rgbl_b200 import _lib as L

SHAPES = {"16x64": [], "8x128": ["-DPOSE_CTAS=8", "-DPOSE_THREADS=128"]}


class EmuPose:
    """rgbl_pose_optimize of an emulated library."""

    def __init__(self, path):
        self.so = C.CDLL(str(path))
        for name, (res, args) in L.SYMBOLS.items():
            fn = getattr(self.so, name)
            fn.restype, fn.argtypes = res, args
        cfg = L.Config(0, 160, 120, 1, 0, 0, L.OrbParams(200, 1.2, 4, 20, 7))
        self.h = C.c_void_p()
        assert self.so.rgbl_create(C.byref(cfg), C.byref(self.h)) == 0

    def __call__(self, pose, xw, obs, inv_s2, stereo, fx, fy, cx, cy, bf):
        pose = np.ascontiguousarray(pose, np.float32); xw = np.ascontiguousarray(xw, np.float32)
        obs = np.ascontiguousarray(obs, np.float32); inv_s2 = np.ascontiguousarray(inv_s2, np.float32)
        stereo = np.ascontiguousarray(stereo, np.uint8)
        n = len(xw)
        out = np.empty(7, np.float32); outlier = np.zeros(max(n, 1), np.uint8); ni = C.c_int(0)
        rc = self.so.rgbl_pose_optimize(self.h, L.ptr(pose), n, L.ptr(xw), L.ptr(obs), L.ptr(inv_s2), L.ptr(stereo), fx, fy, cx, cy, bf,
                                        L.ptr(out), L.ptr(outlier), C.byref(ni))
        assert rc == 0, self.so.rgbl_last_error(self.h)
        return ni.value, out, outlier[:n]

    def close(self):
        self.so.rgbl_destroy(self.h)


@pytest.fixture(scope="module", params=list(SHAPES))
def emu(request):
    e = EmuPose(build.build_full(defines=SHAPES[request.param]))
    yield e
    e.close()


def _subset():
    # n = 3 and 10, past the shared-memory cache (8193, and 20000 where most edges are), a sincos start, rounds ending unconverged
    # (two of them with accepted trials w >= 5), >= 9 rejections ending in qmax == 10, all outliers (H = 0 rounds), the quaternion
    # branches, an edge on the camera plane and bf = 0; the cases of pose_cases.py themselves, picked by name
    want = {"n3", "n10", "n8193", "n20000", "far3", "rej0", "unconv0", "unconv1", "unconv2", "unconv3", "allout", "quat0", "quat3", "plane1",
            "stereo_bf0"}
    return [c for c in PC.all_cases() if c["name"] in want]


CASES = _subset()


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_pose_kernel_emulated(emu, c):
    p = c["problem"]
    ref = PC.reference(p)
    PC.check_coverage(c, ref[3])
    got = emu(*PC.args(p))
    PC.compare(c, got, ref)
    again = emu(*PC.args(p))
    assert again[0] == got[0] and again[1].tobytes() == got[1].tobytes() and again[2].tobytes() == got[2].tobytes()


def test_families_reach_their_paths():
    """Through the oracle's trace, at full size: the families of pose_cases.py reach what they exist for (the per-case expectations,
    and over all cases: a case on the exact bar with a run of >= 9 rejected trials, a qmax == 10 termination and an accepted trial
    w >= 5, a step with theta^2 >= 0.25, a round without an active edge, n past the shared-memory cache, both sides of the n < 10
    break)."""
    traces = {}
    for c in PC.all_cases():
        tr = PC.reference(c["problem"])[3]
        PC.check_coverage(c, tr)
        traces[c["name"]] = (len(c["problem"]["xw"]), tr)
    exact = [t for _, t in traces.values() if PC.qualifies(t)]
    assert any(t["max_reject_run"] >= 9 and t["term_qmax"] >= 1 and t["max_accepted_trial"] >= 5 for t in exact)
    assert any(t["any_sincos"] for _, t in traces.values())
    assert any(t["empty_rounds"] for _, t in traces.values())
    assert max(n for n, _ in traces.values()) > 16 * 512
    assert traces["n9"][1]["rounds"] == 1 and traces["n10"][1]["rounds"] == 4

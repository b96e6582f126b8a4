"""pose_optimize_kernel under the CUDA-on-CPU shim reproduces, byte for byte, what the kernel of commit a3598bb (the last one that built
every LM iteration's system in a pass of its own) computed: inlier count, float32 pose and outlier flags.  The kernel builds the next
system inside the trial evaluation and the classification passes with the same expressions and summation orders as those separate
passes, so nothing may move, not even in the last bit.

Each emulated call costs seconds, so the cases are the ones of pose_cases.py that reach what the fused passes change: runs of
rejected trials whose systems are dropped and accepted trials w >= 5 (rej0, unconv2), rounds with no active edge and the rho == 0 stop
(allout), both sides of the n < 10 break that skips the next round's system (n9, n10), NaN errors from an edge on the camera plane
(plane1), sincos steps (far1) and a grid-stride remainder (n1025); the first three also at 8 x 128.
tests/golden/make_pose_kernel_golden.py wrote tests/golden/pose_kernel_base.npz from that commit's kernel."""
from pathlib import Path

import numpy as np
import pytest

import pose_cases as PC
from cuda_emu import build
from test_cuda_emu_pose import SHAPES, EmuPose

GOLD = Path(__file__).resolve().parent / "golden" / "pose_kernel_base.npz"
CASES = {c["name"]: c for c in PC.all_cases()}
CHECKED = [("16x64", n) for n in ("rej0", "unconv2", "allout", "n9", "n10", "plane1", "far1", "n1025")] + \
          [("8x128", n) for n in ("rej0", "unconv2", "plane1")]


def outputs(e, c):
    """(n_inliers, pose, outlier flags) of the emulated kernel for case c, as the arrays stored in the golden file."""
    ni, pose, out = e(*PC.args(c["problem"]))
    return np.array([ni], np.int32), pose, out


def emulated(shape):
    return EmuPose(build.build_full(defines=SHAPES[shape]))


@pytest.fixture(scope="module")
def emu():
    libs = {}

    def get(shape):
        if shape not in libs:
            libs[shape] = emulated(shape)
        return libs[shape]
    yield get
    for e in libs.values():
        e.close()


@pytest.mark.parametrize("shape,name", CHECKED, ids=[f"{s}-{n}" for s, n in CHECKED])
def test_pose_kernel_matches_base_bitwise(emu, shape, name):
    gold = np.load(GOLD)
    for key, got in zip(("n_inliers", "pose", "outlier"), outputs(emu(shape), CASES[name])):
        want = gold[f"{shape}/{name}/{key}"]
        assert got.dtype == want.dtype and got.shape == want.shape, (key, got.dtype, got.shape, want.dtype, want.shape)
        assert got.tobytes() == want.tobytes(), (shape, name, key)

"""Generates tests/golden/pose_kernel_base.npz: the outputs of pose_optimize_kernel under the CUDA-on-CPU shim (tests/cuda_emu) for the
(cluster shape, case) pairs that tests/test_cuda_emu_pose_bitwise.py checks, keyed "<shape>/<case>/<n_inliers|pose|outlier>".
Run from the repo root of the commit whose kernel is the reference (see that test's docstring)."""
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[2]
sys.path.insert(0, str(ROOT)); sys.path.insert(0, str(ROOT / "tests"))
import test_cuda_emu_pose_bitwise as TB  # noqa: E402

mod = TB._build_module()
libs, out = {}, {}
for shape, name in TB.CHECKED:
    if shape not in libs:
        libs[shape] = TB.emulated(mod, shape)
    for key, a in zip(("n_inliers", "pose", "outlier"), TB.outputs(libs[shape], TB.CASES[name])):
        out[f"{shape}/{name}/{key}"] = a
for e in libs.values():
    e.close()
np.savez_compressed(TB.GOLD, **out)
print(TB.GOLD, TB.GOLD.stat().st_size, "bytes,", len(out), "arrays")

"""Frame::UndistortKeyPoints / ComputeImageBounds of a distorted camera on the CUDA-on-CPU shim (tests/cuda_emu): undistort_keypoints_kernel
through its launcher and the host bounds helper of rgbl_set_camera_distortion, bit for bit against the oracle, with 4 and 5 coefficients."""
import ctypes as C
import importlib.util
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import undistort as U
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import synthetic as S

HERE = Path(__file__).resolve().parent
CAM = (S.TUM1_FX, S.TUM1_FY, S.TUM1_CX, S.TUM1_CY)
DISTS = {"tum1": S.TUM1_DIST, "tum1_4": S.TUM1_DIST[:4], "barrel": np.array([-0.31, 0.11, 0.0012, -0.0021, -0.02], np.float32)}


@pytest.fixture(scope="module")
def emu():
    spec = importlib.util.spec_from_file_location("cuda_emu_build", HERE / "cuda_emu" / "build.py")
    mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
    d = mod.BUILD / "undistort"
    d.mkdir(parents=True, exist_ok=True)
    for f in mod.CSRC.iterdir():
        if f.suffix in (".h", ".cuh", ".inc"):
            (d / f.name).write_text(mod._transform(f.read_text()))
    (d / "depth_kernels.emu.cpp").write_text(mod._transform((mod.CSRC / "depth_kernels.cu").read_text()))
    lib = d / "libcuda_emu_undistort.so"
    subprocess.run(["g++", "-std=c++20", "-O1", "-g", "-pthread", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes",
                    f"-I{HERE / 'cuda_emu'}", f"-I{d}", "-o", str(lib), str(HERE / "cuda_emu" / "emu_undistort.cpp"),
                    str(HERE / "cuda_emu" / "emu_runtime.cpp")], check=True)
    L_ = C.CDLL(str(lib))
    f, i, vp = C.c_float, C.c_int, C.c_void_p
    L_.emu_undistort_keypoints.argtypes = [f, f, f, f, vp, i, vp, vp, i, i, vp]
    L_.emu_image_bounds.argtypes = [f, f, f, f, vp, i, i, i, vp]
    return L_


def _keypoints(rng, n, W, H):
    k = np.zeros(n, L.KP_DTYPE)
    k["x"] = rng.uniform(-25, W + 25, n).astype(np.float32); k["y"] = rng.uniform(-25, H + 25, n).astype(np.float32)
    k["size"] = 31.0; k["angle"] = rng.uniform(0, 360, n); k["response"] = rng.uniform(0, 100, n)
    k["octave"] = rng.integers(0, 8, n); k["class_id"] = -1
    k[:4]["x"] = [0, S.TUM_W, 0, S.TUM_W]; k[:4]["y"] = [0, 0, S.TUM_H, S.TUM_H]
    return k


@pytest.mark.parametrize("name", list(DISTS))
def test_undistort_kernel_device_path(emu, name):
    dist = np.ascontiguousarray(DISTS[name])
    rng = np.random.default_rng(len(name))
    cap, n_kp = 3000, np.array([2999, 1234, 0], np.int32)
    kps = np.zeros((3, cap), L.KP_DTYPE)
    for f in range(3):
        kps[f, :n_kp[f]] = _keypoints(rng, int(n_kp[f]), S.TUM_W, S.TUM_H) if n_kp[f] else kps[f, :0]
    out = np.zeros((3, cap), L.KP_DTYPE); out["class_id"] = 7
    emu.emu_undistort_keypoints(*CAM, L.ptr(dist), len(dist), L.ptr(kps), L.ptr(n_kp), cap, 3, L.ptr(out))
    for f in range(3):
        n = n_kp[f]
        ref = U.undistort_keypoints(kps[f, :n], CAM, dist)
        assert out[f, :n].tobytes() == ref.tobytes(), f              # pt replaced, every other field copied
        assert (out[f, n:]["class_id"] == 7).all()                      # nothing written past n_kp


@pytest.mark.parametrize("name", list(DISTS) + ["k1_zero"])
def test_bounds_host_helper(emu, name):
    dist = np.ascontiguousarray(DISTS.get(name, np.array([0.0, -0.95, 0.004, 0.002, 1.1], np.float32)))
    b = np.empty(4, np.float32)
    emu.emu_image_bounds(*CAM, L.ptr(dist), len(dist), S.TUM_W, S.TUM_H, L.ptr(b))
    assert b.tobytes() == U.image_bounds(S.TUM_W, S.TUM_H, CAM, dist).tobytes()
    if name == "k1_zero":
        assert list(b) == [0, S.TUM_W, 0, S.TUM_H]

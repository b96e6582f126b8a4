"""The stereo rectification kernels (stereo_kernels.cu: the conversion of the float maps into OpenCV's fixed-point form and the batched
remap of both cameras' frames) on the CUDA-on-CPU shim (tests/cuda_emu), bit for bit against the oracle (oracle/remap_oracle.cpp, pinned
to cv2 in tests/test_oracle_rectify.py): both cameras and several frames per camera in one launch, maps past every edge, wholly outside
the image, exact 1/64 ties and saturating values, an odd width (a partial last group of 4 pixels) and the last row and column."""
import ctypes as C
import importlib.util
import subprocess
from pathlib import Path

import numpy as np
import pytest

from oracle import _p
from oracle import rectify as RC

HERE = Path(__file__).resolve().parent


@pytest.fixture(scope="module")
def emu():
    spec = importlib.util.spec_from_file_location("cuda_emu_build", HERE / "cuda_emu" / "build.py")
    mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
    d = mod.BUILD / "rectify"
    d.mkdir(parents=True, exist_ok=True)
    for f in mod.CSRC.iterdir():
        if f.suffix in (".h", ".cuh", ".inc"):
            (d / f.name).write_text(mod._transform(f.read_text()))
    (d / "stereo_kernels.emu.cpp").write_text(mod._transform((mod.CSRC / "stereo_kernels.cu").read_text()))
    lib = d / "libcuda_emu_rectify.so"
    subprocess.run(["g++", "-std=c++20", "-O1", "-g", "-pthread", "-fPIC", "-shared", "-ffp-contract=off", "-Wno-unknown-pragmas", "-Wno-attributes",
                    f"-I{HERE / 'cuda_emu'}", f"-I{d}", "-o", str(lib), str(HERE / "cuda_emu" / "emu_rectify.cpp"),
                    str(HERE / "cuda_emu" / "emu_runtime.cpp")], check=True)
    L_ = C.CDLL(str(lib))
    L_.emu_rectify_maps.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    L_.emu_rectify.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int]
    return L_


def edge_maps(rng, W, H):
    """float32 maps over the image and beyond every edge, with rows of exact 1/64 ties, rows wholly outside the image, saturating
    values, and the last row / column sampled exactly"""
    mx = rng.uniform(-3, W + 2, (H, W)).astype(np.float32)
    my = rng.uniform(-3, H + 2, (H, W)).astype(np.float32)
    mx[1] = np.round(mx[1] * 64) / 64; my[1] = np.round(my[1] * 64) / 64
    mx[2] = rng.uniform(-1e4, -2, W); my[3] = rng.uniform(H + 1, 1e4, W)                      # wholly outside
    sat = np.array([1e6, -1e6, 1e9, -1e9, 3e38, -3e38, -3e38, 3e38], np.float32)
    mx[4, :8] = sat; my[4, :8] = sat[::-1]
    mx[5] = W - 1; my[5] = np.arange(W, dtype=np.float32) % H                                   # last column
    my[6] = H - 1; mx[6] = np.arange(W, dtype=np.float32)                                       # last row
    mx[7] = W - 1 + np.float32(1 / 64); my[7] = H - 1 - np.float32(31 / 64)                    # taps just past the last column
    return mx, my


@pytest.mark.parametrize("W,H", [(97, 61), (64, 33)])
def test_rectify_kernels_match_oracle(emu, W, H):
    rng = np.random.default_rng(W * H)
    n = 3                                                       # frames per camera: 2 n raw planes in one launch
    m1l, m2l = edge_maps(rng, W, H)
    m1r, m2r = edge_maps(rng, W, H)
    maps = np.ascontiguousarray(np.stack([m1l, m2l, m1r, m2r]))
    pitch = (W + 3) & ~3
    xy = np.full((2, H, pitch), 0xDEADBEEF, np.uint32); a = np.full((2, H, pitch), 0xBEEF, np.uint16)
    emu.emu_rectify_maps(_p(maps), W, H, _p(xy), _p(a), pitch)
    for cam, (mx, my) in enumerate(((m1l, m2l), (m1r, m2r))):
        rxy, ra = RC.convert_maps(mx, my)
        got = xy[cam, :, :W]
        assert ((got & 0xFFFF).astype(np.uint16).view(np.int16) == rxy[..., 0]).all(), cam
        assert ((got >> 16).astype(np.uint16).view(np.int16) == rxy[..., 1]).all(), cam
        assert (a[cam, :, :W] == ra).all(), cam
    src_pitch = (W + 63) & ~63
    raw = rng.integers(0, 256, (2 * n, H, src_pitch), dtype=np.uint8)
    raw[0] = 255                                                # saturation of the weighted sum
    dst_pitch, dst_off = src_pitch, 128
    stride = dst_off + dst_pitch * H + 64
    dst = np.full((2 * n, stride), 7, np.uint8)
    emu.emu_rectify(_p(xy), _p(a), pitch, W, H, _p(raw), src_pitch, _p(dst), stride, dst_off, dst_pitch, n)
    for s in range(2 * n):
        mx, my = (m1l, m2l) if s < n else (m1r, m2r)
        ref = RC.remap(np.ascontiguousarray(raw[s, :, :W]), mx, my)
        img = dst[s, dst_off:dst_off + dst_pitch * H].reshape(H, dst_pitch)
        assert (img[:, :W] == ref).all(), (s, int((img[:, :W] != ref).sum()))
        assert (img[:, W:] == 7).all() and (dst[s, :dst_off] == 7).all() and (dst[s, dst_off + dst_pitch * H:] == 7).all()   # nothing else written
    assert (RC.remap(np.ascontiguousarray(raw[0, :, :W]), m1l, m2l) == 255).any()

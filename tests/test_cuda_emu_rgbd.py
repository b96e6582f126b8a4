"""The RGB-D device code paths on the CUDA-on-CPU shim (tests/cuda_emu): the 16-bit depth PNG reconstruction (png_unfilter_gray_kernel's
depth output stage, an image taller than one 512-row band) and the uint16 depth gather (depth_gather_kernel<uint16_t>), against the oracle."""
import ctypes as C

import numpy as np
import pytest

import oracle
from cuda_emu import build
from oracle import rgbd as R
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import synthetic as S


@pytest.fixture(scope="module")
def emu():
    L_ = C.CDLL(str(build.build_full()))
    L_.emu_png_depth16.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p]
    L_.emu_gather_u16.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_int, C.c_float, C.c_void_p, C.c_void_p]
    return L_


def test_depth16_png_kernel_device_path(emu):
    rng = np.random.default_rng(12)
    w, h = 37, 600                                   # two bands of 512 rows, odd width (last uint16 of a row written alone)
    u = rng.integers(0, 65536, (h, w)).astype(np.uint16)
    u[100:300, 5:20] = 0
    for filters in (None, rng.integers(0, 5, h)):
        png = S.encode_png16(u, filters, 5000)
        ref = R.png_decode_depth16(png)
        assert (ref == u).all()
        out = np.empty((h, w), np.uint16)
        buf = np.frombuffer(png, np.uint8)
        assert emu.emu_png_depth16(L.ptr(buf), len(buf), w, h, L.ptr(out)) == 0
        assert (out == ref).all()


def test_depth16_png_kernel_rejects_8bit(emu):
    png = S.encode_png(np.zeros((20, 30), np.uint8))
    buf = np.frombuffer(png, np.uint8)
    out = np.empty((20, 30), np.uint16)
    assert emu.emu_png_depth16(L.ptr(buf), len(buf), 30, 20, L.ptr(out)) == -2


@pytest.mark.parametrize("factor", [1, 256, 5000])
def test_uint16_gather_device_path(emu, factor):
    seq = S.PlaneSequence(9, 2, W=300, H=160)
    img, dep = seq.image(1), seq.depth16(1, factor, 0.2)
    if factor == 1:
        dep = np.where(dep > 0, np.random.default_rng(2).integers(1, 65536, dep.shape), 0).astype(np.uint16)      # the whole range, holes kept
    ex = oracle.Extractor(500)
    scale = R.depth_map_factor(factor)
    fr = R.rgbd_frame(ex, img, dep, scale, S.KITTI_BF)
    k = np.ascontiguousarray(fr["k"])
    n = len(k)
    d = np.empty(n, np.float32); ur = np.empty(n, np.float32)
    emu.emu_gather_u16(L.ptr(dep), dep.shape[1], dep.shape[0], float(scale), L.ptr(k), n, S.KITTI_BF, L.ptr(d), L.ptr(ur))
    assert (d.view(np.uint32) == fr["depth"].view(np.uint32)).all() and (ur.view(np.uint32) == fr["ur"].view(np.uint32)).all()
    assert (fr["depth"] < 0).any() and (fr["depth"] > 0).sum() > n // 2

"""The input-resize kernels on the CUDA-on-CPU shim (tests/cuda_emu): launch_resize_planes (orb_kernels.cu: the pyramid's resize kernels
reading separate source planes, staged-tile form up to a ratio of about 1.35, gather form above) and launch_resize_depth16 (depth_kernels.cu),
several planes per launch.  Whole output planes must equal cv2.resize(INTER_LINEAR) - or, without cv2, the oracle pinned to it in
tests/test_oracle_resize.py - bit for bit, and nothing outside the destination images may be written."""
import ctypes as C

import numpy as np
import pytest

import resize_oracle as RO
from cuda_emu import build
from oracle import _p


@pytest.fixture(scope="module")
def emu():
    L_ = C.CDLL(str(build.build_full()))
    L_.emu_resize_planes.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int]
    L_.emu_resize_depth16.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int]
    return L_


def reference(src, dw, dh):
    try:
        import cv2
        return cv2.resize(src, (dw, dh), interpolation=cv2.INTER_LINEAR)
    except ImportError:
        return RO.resize_linear(src, dw, dh)


def tile_form(sw, sh, dw, dh):
    """the launcher's choice: the staged-tile kernel when the source rectangle of a 128 x 16 tile fits its 24 x 192-byte stage"""
    return (sw / dw) * 127 + 18 <= 191 and (sh / dh) * 15 + 3 <= 24


# ratios on both sides of the tile / gather switch, odd sizes, aspect changes, a partial last group of 4 pixels
U8 = [((150, 97), (125, 81)), ((161, 99), (130, 80)), ((200, 120), (100, 60)), ((203, 77), (101, 70)), ((257, 130), (97, 41)), ((96, 64), (93, 61))]


@pytest.mark.parametrize("src_size,dst_size", U8)
def test_resize_planes_match_cv2(emu, src_size, dst_size):
    (sw, sh), (dw, dh) = src_size, dst_size
    rng = np.random.default_rng(sw * dh)
    n = 3
    spitch, dpitch, off = (sw + 63) & ~63, (dw + 63) & ~63, 128
    src = rng.integers(0, 256, (n, sh, spitch), dtype=np.uint8)
    stride = off + dpitch * dh + 64
    dst = np.full((n, stride), 7, np.uint8)
    emu.emu_resize_planes(_p(src), sw, sh, spitch, _p(dst), stride, off, dw, dh, dpitch, n)
    for f in range(n):
        ref = reference(np.ascontiguousarray(src[f, :, :sw]), dw, dh)
        img = dst[f, off:off + dpitch * dh].reshape(dh, dpitch)
        assert (img[:, :dw] == ref).all(), (f, int((img[:, :dw] != ref).sum()))
        assert (dst[f, :off] == 7).all() and (dst[f, off + dpitch * dh:] == 7).all()


def test_cases_cover_both_kernel_forms():
    forms = {tile_form(*s, *d) for s, d in U8}
    assert forms == {True, False}


@pytest.mark.parametrize("src_size,k", [((160, 120), (2, 2)), ((99, 63), (3, 3)), ((128, 96), (4, 4)), ((128, 90), (2, 3)), ((90, 64), (1, 2)),
                                        ((66, 48), (3, 1))])
def test_resize_depth16_matches_cv2(emu, src_size, k):
    (sw, sh), (kx, ky) = src_size, k
    dw, dh = sw // kx, sh // ky
    rng = np.random.default_rng(sw + 7 * sh)
    n = 2
    spitch, dpitch = ((sw * 2 + 63) // 64) * 32, ((dw * 2 + 63) // 64) * 32
    src = rng.integers(0, 65536, (n, sh, spitch), dtype=np.uint16)
    src[1][rng.random((sh, spitch)) < 0.2] = 0                          # a depth image with holes
    src[0, 0, :sw] = 65535; src[0, 1, :sw] = 65534                      # the top of the value range
    dst = np.full((n, dh, dpitch), 7, np.uint16)
    emu.emu_resize_depth16(_p(src), sh, spitch, kx, ky, _p(dst), dw, dh, dpitch, n)
    for f in range(n):
        ref = reference(np.ascontiguousarray(src[f, :, :sw]), dw, dh)
        assert (dst[f, :, :dw] == ref).all(), (f, int((dst[f, :, :dw] != ref).sum()))
        assert (dst[f, :, dw:] == 7).all()

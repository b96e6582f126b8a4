"""The colour-input kernels on the CUDA-on-CPU shim (tests/cuda_emu), through their launchers, bit for bit against cv2 (or, without cv2,
the per-channel oracles pinned to it in tests/test_oracle_colour.py followed by cvtColor's fixed-point formula): the gray conversion of
3- and 4-channel planes (orb_kernels.cu gray_planes_kernel), the input resize of colour planes in its staged-tile and gather forms
(resize_level_kernel / resize_level_gather_kernel with CH = 3, 4), the stereo remap of colour planes (stereo_kernels.cu rectify_kernel
with CH = 3, 4) and the PNG reconstruction into colour planes (png_kernels.cu).  Several planes per launch, odd sizes with a partial last
group of 4 pixels, both channel orders; nothing outside the destination images may be written."""
import ctypes as C

import numpy as np
import pytest

import resize_oracle as RO
from cuda_emu import build
from oracle import _p
from oracle import rectify as RC
from orb_slam3_rgbl_b200 import synthetic as S

RED, BLUE = 9798, 3735          # the weight of channel 0: Camera.RGB = 1 (RGB2GRAY) / 0 (BGR2GRAY)


@pytest.fixture(scope="module")
def emu():
    L_ = C.CDLL(str(build.build_full()))
    i, vp, sz = C.c_int, C.c_void_p, C.c_size_t
    L_.emu_gray_planes.argtypes = [vp, i, i, i, i, i, vp, sz, i, i, i]
    L_.emu_resize_colour.argtypes = [vp, i, i, i, i, i, vp, sz, i, i, i, i, i]
    L_.emu_rectify_colour.argtypes = [vp, i, i, vp, i, i, i, i, i, vp, sz, i, i, i]
    L_.emu_png_pixels.argtypes = [i, vp, vp, i, i, vp, sz, i]
    return L_


def to_gray(img, w0):
    """cvtColor({RGB,BGR,RGBA,BGRA}2GRAY) of an H x W x C image whose channel 0 has the weight w0"""
    try:
        import cv2
        code = {(3, RED): cv2.COLOR_RGB2GRAY, (3, BLUE): cv2.COLOR_BGR2GRAY, (4, RED): cv2.COLOR_RGBA2GRAY, (4, BLUE): cv2.COLOR_BGRA2GRAY}
        return cv2.cvtColor(np.ascontiguousarray(img), code[(img.shape[2], w0)])
    except ImportError:
        c = img.astype(np.int64)
        return ((c[..., 0] * w0 + c[..., 1] * 19235 + c[..., 2] * (RED + BLUE - w0) + (1 << 14)) >> 15).astype(np.uint8)


def resize(img, w, h):
    try:
        import cv2
        return cv2.resize(np.ascontiguousarray(img), (w, h), interpolation=cv2.INTER_LINEAR)
    except ImportError:
        return np.stack([RO.resize_linear(np.ascontiguousarray(img[..., k]), w, h) for k in range(img.shape[2])], -1)


def remap(img, mx, my):
    try:
        import cv2
        return cv2.remap(np.ascontiguousarray(img), mx, my, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    except ImportError:
        return np.stack([RC.remap(np.ascontiguousarray(img[..., k]), mx, my) for k in range(img.shape[2])], -1)


def planes(rng, n, w, h, ch):
    """n colour planes of w x h pixels in rows padded to 64 bytes -> (planes [n][h][pitch], pitch)"""
    pitch = (w * ch + 63) & ~63
    return rng.integers(0, 256, (n, h, pitch), dtype=np.uint8), pitch


def image(p, w, ch):
    return np.ascontiguousarray(p[:, :w * ch].reshape(p.shape[0], w, ch))


def dst_buffer(n, w, h, off=128):
    """destination planes of dst_stride bytes, image at `off`, 64-byte rows, everything else 7"""
    dpitch = (w + 63) & ~63
    stride = off + dpitch * h + 64
    return np.full((n, stride), 7, np.uint8), stride, off, dpitch


def check_dst(dst, f, off, dpitch, w, h, want, padding=False):
    """padding: the kernel may write its last 32-bit word into the rows' padding, as the pyramid's resize kernels do"""
    img = dst[f, off:off + dpitch * h].reshape(h, dpitch)
    assert (img[:, :w] == want).all(), (f, int((img[:, :w] != want).sum()))
    assert (img[:, (w + 3) & ~3 if padding else w:] == 7).all()
    assert (dst[f, :off] == 7).all() and (dst[f, off + dpitch * h:] == 7).all()           # nothing else written


@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("w0", [RED, BLUE], ids=["rgb", "bgr"])
@pytest.mark.parametrize("w,h", [(97, 61), (128, 33), (21, 7)])
def test_gray_planes_match_cvtcolor(emu, ch, w0, w, h):
    rng = np.random.default_rng(w * h + ch + w0)
    n = 3
    src, spitch = planes(rng, n, w, h, ch)
    src[0, 0, :ch * 4] = 255                                    # the top of the range
    dst, stride, off, dpitch = dst_buffer(n, w, h)
    emu.emu_gray_planes(_p(src), w, h, spitch, ch, w0, _p(dst), stride, off, dpitch, n)
    for f in range(n):
        check_dst(dst, f, off, dpitch, w, h, to_gray(image(src[f], w, ch), w0))


def tile_form(sw, sh, dw, dh):
    """the launcher's choice: the staged-tile kernel when the source rectangle of a 128 x 16 tile fits its stage (for any channel count)"""
    return (sw / dw) * 127 + 18 <= 191 and (sh / dh) * 15 + 3 <= 24


# ratios on both sides of the tile / gather switch, odd sizes, the factor-2 case, a partial last group of 4 pixels
SIZES = [((150, 97), (125, 81)), ((203, 77), (101, 70)), ((200, 120), (100, 60)), ((257, 130), (97, 41)), ((96, 64), (93, 61))]


def test_resize_cases_cover_both_kernel_forms():
    assert {tile_form(*s, *d) for s, d in SIZES} == {True, False}


@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("w0", [RED, BLUE], ids=["rgb", "bgr"])
@pytest.mark.parametrize("src_size,dst_size", SIZES)
def test_resize_colour_matches_cv2(emu, ch, w0, src_size, dst_size):
    (sw, sh), (dw, dh) = src_size, dst_size
    rng = np.random.default_rng(sw * dh + ch)
    n = 3
    src, spitch = planes(rng, n, sw, sh, ch)
    dst, stride, off, dpitch = dst_buffer(n, dw, dh)
    emu.emu_resize_colour(_p(src), sw, sh, spitch, ch, w0, _p(dst), stride, off, dw, dh, dpitch, n)
    for f in range(n):
        check_dst(dst, f, off, dpitch, dw, dh, to_gray(resize(image(src[f], sw, ch), dw, dh), w0), padding=True)


def edge_maps(rng, W, H, sw, sh):
    """float32 maps over the source and past every edge, rows wholly outside, exact 1/64 ties, the last row and column"""
    mx = rng.uniform(-3, sw + 2, (H, W)).astype(np.float32)
    my = rng.uniform(-3, sh + 2, (H, W)).astype(np.float32)
    mx[1] = np.round(mx[1] * 64) / 64; my[1] = np.round(my[1] * 64) / 64
    mx[2] = rng.uniform(-1e4, -2, W); my[3] = rng.uniform(sh + 1, 1e4, W)
    mx[4] = sw - 1; my[4] = np.arange(W, dtype=np.float32) % sh
    my[5] = sh - 1; mx[5] = np.arange(W, dtype=np.float32) % sw
    return mx, my


@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("w0", [RED, BLUE], ids=["rgb", "bgr"])
@pytest.mark.parametrize("W,H,sw,sh", [(97, 61, 97, 61), (64, 33, 80, 41)], ids=["same_size", "input_size"])
def test_rectify_colour_matches_cv2(emu, ch, w0, W, H, sw, sh):
    rng = np.random.default_rng(W * H + ch + w0)
    n = 2                                                       # pairs: 2 n raw planes in one launch
    m1l, m2l = edge_maps(rng, W, H, sw, sh)
    m1r, m2r = edge_maps(rng, W, H, sw, sh)
    maps = np.ascontiguousarray(np.stack([m1l, m2l, m1r, m2r]))
    src, spitch = planes(rng, 2 * n, sw, sh, ch)
    dst, stride, off, dpitch = dst_buffer(2 * n, W, H)
    emu.emu_rectify_colour(_p(maps), W, H, _p(src), sw, sh, spitch, ch, w0, _p(dst), stride, off, dpitch, n)
    for s in range(2 * n):
        mx, my = (m1l, m2l) if s < n else (m1r, m2r)
        check_dst(dst, s, off, dpitch, W, H, to_gray(remap(image(src[s], sw, ch), mx, my), w0))


@pytest.mark.parametrize("ch", [3, 4])
@pytest.mark.parametrize("w,h", [(97, 61), (40, 600)])          # 600 rows: two bands of the wavefront
def test_png_pixels_are_the_files_samples(emu, ch, w, h):
    n = 2
    imgs = [S.colorize(S.make_image(5 + f, w, h, 20), seed=f, alpha=ch == 4) for f in range(n)]
    bufs = [np.frombuffer(S.encode_png(i), np.uint8) for i in imgs]
    pa = (C.c_void_p * n)(*[b.ctypes.data for b in bufs]); sizes = (C.c_size_t * n)(*[len(b) for b in bufs])
    pitch = (w * ch + 63) & ~63
    stride = pitch * h + 64
    dst = np.full((n, stride), 7, np.uint8)
    assert emu.emu_png_pixels(n, pa, sizes, w, h, _p(dst), stride, pitch) == ch
    for f in range(n):
        got = dst[f, :pitch * h].reshape(h, pitch)
        assert (got[:, :w * ch] == imgs[f].reshape(h, w * ch)).all(), f
        assert (got[:, w * ch:] == 7).all() and (dst[f, pitch * h:] == 7).all()

"""The claim the colour input rests on: OpenCV's colour resize / remap followed by cvtColor equals the per-channel 8-bit restatements the
device kernels follow (oracle.resize_linear, the pyramid's fixed-point cv::resize; oracle.rectify.remap, oracle/remap_oracle.cpp)
followed by cvtColor's fixed-point formula (9798 R + 19235 G + 3735 B + 2^14) >> 15, alpha ignored.  3 and 4 channels, both channel orders
(RGB2GRAY / BGR2GRAY: channel 0 weighted as red or as blue), odd sizes, both forms of the device resize (ratios below and above the
staged tile's limit, the factor-2 case) and maps with taps outside the source.  Live when cv2 is importable, and through the committed
tests/golden/colour_golden.npz (written by tests/golden/make_colour_golden.py) in any case."""
from pathlib import Path

import numpy as np
import pytest

import oracle
from oracle import rectify as RC

GOLD = Path(__file__).resolve().parent / "golden" / "colour_golden.npz"
RED, BLUE = 9798, 3735

# (source w, h) -> (destination w, h): tile-form ratios, gather-form ratios, factor 2, odd sizes
RESIZE = [((150, 97), (125, 81)), ((203, 77), (101, 70)), ((200, 120), (100, 60)), ((257, 130), (97, 41)), ((96, 64), (93, 61)),
          ((191, 109), (64, 36)), ((120, 50), (40, 20))]
REMAP = [((97, 61), (97, 61)), ((80, 41), (64, 33))]        # (source w, h), (map w, h)
GOLD_MAX_PIXELS = 15000          # the golden file keeps the small cases (the others are checked live)


def gray(img, w0):
    """cvtColor's formula with channel 0 weighted w0 (RED: RGB2GRAY, BLUE: BGR2GRAY)"""
    c = img.astype(np.int64)
    return ((c[..., 0] * w0 + c[..., 1] * 19235 + c[..., 2] * (RED + BLUE - w0) + (1 << 14)) >> 15).astype(np.uint8)


def per_channel(fn, img):
    return np.stack([fn(np.ascontiguousarray(img[..., k])) for k in range(img.shape[2])], -1)


def _maps(rng, W, H, sw, sh):
    mx = rng.uniform(-3, sw + 2, (H, W)).astype(np.float32)
    my = rng.uniform(-3, sh + 2, (H, W)).astype(np.float32)
    mx[1] = np.round(mx[1] * 64) / 64; my[1] = np.round(my[1] * 64) / 64
    mx[2] = rng.uniform(-1e4, -2, W); my[3] = rng.uniform(sh + 1, 1e4, W)
    return mx, my


def cases():
    """name, kind, image, (dw, dh) or (mapx, mapy), w0"""
    out = []
    for i, ((sw, sh), (dw, dh)) in enumerate(RESIZE):
        for ch in (3, 4):
            rng = np.random.default_rng(200 + 10 * i + ch)
            w0 = RED if (i + ch) % 2 else BLUE
            out.append((f"resize_{sw}x{sh}_{dw}x{dh}_{ch}", "resize", rng.integers(0, 256, (sh, sw, ch), dtype=np.uint8), (dw, dh), w0))
    for i, ((sw, sh), (W, H)) in enumerate(REMAP):
        for ch in (3, 4):
            rng = np.random.default_rng(300 + 10 * i + ch)
            w0 = BLUE if (i + ch) % 2 else RED
            out.append((f"remap_{sw}x{sh}_{W}x{H}_{ch}", "remap", rng.integers(0, 256, (sh, sw, ch), dtype=np.uint8), _maps(rng, W, H, sw, sh), w0))
    return out


def cv2_result(kind, img, arg, w0):
    import cv2
    out = cv2.resize(img, arg, interpolation=cv2.INTER_LINEAR) if kind == "resize" else \
        cv2.remap(img, arg[0], arg[1], cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    code = {(3, RED): cv2.COLOR_RGB2GRAY, (3, BLUE): cv2.COLOR_BGR2GRAY, (4, RED): cv2.COLOR_RGBA2GRAY, (4, BLUE): cv2.COLOR_BGRA2GRAY}
    return cv2.cvtColor(out, code[(img.shape[2], w0)])


def oracle_result(kind, img, arg, w0):
    fn = (lambda p: oracle.resize_linear(p, *arg)) if kind == "resize" else (lambda p: RC.remap(p, *arg))
    return gray(per_channel(fn, img), w0)


CASES = cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_per_channel_oracle_then_gray_equals_cv2_live(case):
    pytest.importorskip("cv2")
    _, kind, img, arg, w0 = case
    assert (oracle_result(kind, img, arg, w0) == cv2_result(kind, img, arg, w0)).all()


def test_per_channel_oracle_then_gray_equals_golden():
    g = np.load(GOLD)
    kept = [c for c in CASES if c[2].shape[0] * c[2].shape[1] <= GOLD_MAX_PIXELS]
    assert {c[1] for c in kept} == {"resize", "remap"} and len({c[2].shape[2] for c in kept}) == 2
    for name, kind, img, arg, w0 in kept:
        assert (g[name + "_src"] == img).all(), name
        assert (oracle_result(kind, img, arg, w0) == g[name + "_cv2"]).all(), name


def test_gray_formula_equals_cvtcolor_on_every_colour():
    cv2 = pytest.importorskip("cv2")
    v = np.arange(1 << 24, dtype=np.uint32)
    img = np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)
    assert (gray(img, RED) == cv2.cvtColor(img, cv2.COLOR_RGB2GRAY)).all()
    assert (gray(img, BLUE) == cv2.cvtColor(img, cv2.COLOR_BGR2GRAY)).all()

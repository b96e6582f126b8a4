"""The oracle's cv::resize(INTER_LINEAR) restatements: oracle.resize_linear (oracle/orb_extractor_oracle.cpp), the pyramid's fixed-point
form for 8-bit images, and resize_oracle.resize_linear_u16 (tests/resize_oracle.py), the float form of OpenCV's 16-bit linear resize,
against python-cv2: live when cv2 is importable, and through the committed tests/golden/resize_golden.npz (written by tests/golden/make_resize_golden.py) in any case.  These are the resizes
System::TrackRGBD and System::TrackStereo run when Settings::needToResize(): 8-bit images at any downscale, 16-bit depth images at integer
factors (the case the device's depth resize restates), including depth images with holes (zeros)."""
from pathlib import Path

import numpy as np
import pytest

import resize_oracle as RO

GOLD = Path(__file__).resolve().parent / "golden" / "resize_golden.npz"

# (source w, h) -> (destination w, h): camera-sized downscales, odd sizes and aspect changes
U8_SHAPES = [((1280, 720), (640, 360)), ((1241, 376), (620, 188)), ((752, 480), (640, 408)), ((1920, 1080), (1241, 698)),
             ((1280, 720), (853, 480)), ((641, 481), (320, 240)), ((1280, 720), (960, 540)), ((97, 61), (48, 30)), ((203, 77), (101, 70)),
             ((64, 40), (63, 13)), ((333, 101), (111, 100)), ((160, 120), (128, 96))]
U16_SHAPES = [((1280, 720), (640, 360)), ((1280, 720), (320, 180)), ((640, 480), (320, 240)), ((1920, 1080), (640, 360)),
              ((1282, 722), (641, 361)), ((1280, 720), (640, 240)), ((640, 480), (640, 240)), ((99, 63), (33, 21)), ((160, 120), (40, 30))]
GOLD_MAX_PIXELS = 40000          # the golden file keeps the small cases (the large ones are checked live)


def _depth_like(rng, w, h):
    """a depth image in millimetres with holes: zeros in blobs and single pixels, a far plane, a near object"""
    d = (800 + 7000 * np.linspace(0, 1, w)[None, :] + rng.integers(0, 400, (h, w))).astype(np.uint16)
    d[h // 4: h // 2, w // 3: w // 2] = rng.integers(300, 900, (h // 2 - h // 4, w // 2 - w // 3))
    d[rng.random((h, w)) < 0.15] = 0
    d[: h // 8, -w // 5:] = 0
    d[-1, :] = 65535
    return d


def cases():
    """name, source image, destination size"""
    out = []
    for i, ((sw, sh), (dw, dh)) in enumerate(U8_SHAPES):
        rng = np.random.default_rng(100 + i)
        out.append((f"u8_{sw}x{sh}_{dw}x{dh}", rng.integers(0, 256, (sh, sw), dtype=np.uint8), dw, dh))
    for i, ((sw, sh), (dw, dh)) in enumerate(U16_SHAPES):
        rng = np.random.default_rng(200 + i)
        out.append((f"u16_{sw}x{sh}_{dw}x{dh}", rng.integers(0, 65536, (sh, sw), dtype=np.uint16), dw, dh))
        out.append((f"u16depth_{sw}x{sh}_{dw}x{dh}", _depth_like(rng, sw, sh), dw, dh))
    return out


def oracle_resize(src, dw, dh):
    return RO.resize_linear(src, dw, dh)


def cv2_resize(src, dw, dh):
    import cv2
    return cv2.resize(src, (dw, dh), interpolation=cv2.INTER_LINEAR)


@pytest.mark.parametrize("name,src,dw,dh", cases(), ids=[c[0] for c in cases()])
def test_oracle_resize_matches_cv2_live(name, src, dw, dh):
    pytest.importorskip("cv2")
    got, ref = oracle_resize(src, dw, dh), cv2_resize(src, dw, dh)
    assert got.dtype == ref.dtype and got.shape == ref.shape == (dh, dw)
    assert (got == ref).all(), (name, int((got != ref).sum()))


def test_oracle_resize_matches_golden():
    g = np.load(GOLD)
    names = [n[:-4] for n in g.files if n.endswith("_src")]
    assert len(names) >= 9 and any(n.startswith("u8_") for n in names) and any(n.startswith("u16depth_") for n in names)
    for n in names:
        src, ref = g[n + "_src"], g[n + "_cv2"]
        got = oracle_resize(src, ref.shape[1], ref.shape[0])
        assert (got == ref).all(), (n, int((got != ref).sum()))
        assert n.startswith("u8_") or ((src == 0).any() if n.startswith("u16depth_") else True)


def test_golden_cases_are_the_small_cases():
    g = np.load(GOLD)
    want = {n for n, src, _, _ in cases() if src.size <= GOLD_MAX_PIXELS}
    assert {n[:-4] for n in g.files if n.endswith("_src")} == want

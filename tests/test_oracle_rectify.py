"""The remap oracle (oracle/remap_oracle.cpp: cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of an 8UC1 image with two CV_32FC1 maps, as
System::TrackStereo rectifies a pair) against python-cv2, live and through tests/golden/remap_golden.npz: an odd size, maps past every edge
and wholly outside the image, exact 1/64 ties, saturating values, the last row and column, and the maps of cv2.stereoRectify +
cv2.initUndistortRectifyMap of a distorted rig with R != I."""
from pathlib import Path

import numpy as np
import pytest

from oracle import rectify as RC

GOLD = Path(__file__).resolve().parent / "golden" / "remap_golden.npz"
W, H = 97, 61


def edge_maps(seed):
    """maps of a W x H output over the image and past every edge, with rows of exact 1/64 ties (both coordinates), rows wholly outside,
    saturating values and exact samples of the last row and column"""
    rng = np.random.default_rng(seed)
    mx = rng.uniform(-4, W + 3, (H, W)).astype(np.float32)
    my = rng.uniform(-4, H + 3, (H, W)).astype(np.float32)
    mx[1] = np.round(mx[1] * 64) / 64; my[1] = np.round(my[1] * 64) / 64
    mx[2] = (np.arange(W) + 0.5 / 32 + np.arange(W) % 4 / 32).astype(np.float32)                  # odd multiples of 1/64
    mx[3] = rng.uniform(-1e4, -2, W); my[4] = rng.uniform(H + 1, 1e4, W)                        # wholly outside
    sat = np.array([1e6, -1e6, 1e9, -1e9, 3e38, -3e38, -3e38, 3e38, 2**26, -2**26], np.float32)
    mx[5, :10] = sat; my[5, :10] = sat[::-1]
    mx[6] = W - 1; my[6] = np.arange(W, dtype=np.float32) % H                                  # last column
    my[7] = H - 1; mx[7] = np.arange(W, dtype=np.float32)                                      # last row
    mx[8] = W - 1 + np.float32(3 / 64); my[8] = H - 1 - np.float32(17 / 64)
    return mx, my


def rig_maps():
    """M1l, M2l, M1r, M2r of cv2.stereoRectify + cv2.initUndistortRectifyMap(CV_32FC1) for a small distorted rig with R != I"""
    import cv2
    K1 = np.array([[60.0, 0, 48.3], [0, 59.5, 30.1], [0, 0, 1]]); K2 = np.array([[61.0, 0, 47.6], [0, 60.2, 30.7], [0, 0, 1]])
    D1 = np.array([-0.28, 0.07, 2e-4, 2e-5]); D2 = np.array([-0.27, 0.068, -1e-4, 3e-5])
    R = cv2.Rodrigues(np.array([0.01, -0.02, 0.005]))[0]; t = np.array([-0.11, 0.001, 0.0005])
    R1, R2, P1, P2, *_ = cv2.stereoRectify(K1, D1, K2, D2, (W, H), R, t, flags=cv2.CALIB_ZERO_DISPARITY, alpha=0)
    m1l, m2l = cv2.initUndistortRectifyMap(K1, D1, R1, P1[:3, :3], (W, H), cv2.CV_32FC1)
    m1r, m2r = cv2.initUndistortRectifyMap(K2, D2, R2, P2[:3, :3], (W, H), cv2.CV_32FC1)
    return m1l, m2l, m1r, m2r


def cases(with_cv2=True):
    """(name, src, mapx, mapy); the rig case needs cv2"""
    rng = np.random.default_rng(5)
    src = rng.integers(0, 256, (H, W), dtype=np.uint8)
    out = [("edges_a", src, *edge_maps(1)), ("edges_b", np.full((H, W), 255, np.uint8), *edge_maps(2))]
    if with_cv2:
        m1l, m2l, m1r, m2r = rig_maps()
        out += [("rig_left", src, m1l, m2l), ("rig_right", src[::-1].copy(), m1r, m2r)]
    return out


def cv2_remap(src, mx, my):
    import cv2
    return cv2.remap(src, mx, my, cv2.INTER_LINEAR)


def test_remap_matches_cv2_live():
    cv2 = pytest.importorskip("cv2")
    for name, src, mx, my in cases():
        assert (RC.remap(src, mx, my) == cv2_remap(src, mx, my)).all(), name
        # the fixed-point form equals cv2.convertMaps(CV_16SC2) wherever map * 32 fits an int (beyond, OpenCV's SIMD conversion does not
        # saturate; every tap of such a pixel lies outside the image either way)
        xy, a = RC.convert_maps(mx, my)
        c1, c2 = cv2.convertMaps(mx, my, cv2.CV_16SC2)
        ok = (np.abs(mx) < 2**26) & (np.abs(my) < 2**26)
        assert (xy[ok] == c1[ok]).all() and (a[ok] == c2[ok]).all(), name


def test_remap_matches_golden():
    g = np.load(GOLD)
    names = {n for n, *_ in cases(with_cv2=False)} | {"rig_left", "rig_right"}
    for name in names:
        src, mx, my = g[name + "_src"], g[name + "_mapx"], g[name + "_mapy"]
        assert (RC.remap(src, mx, my) == g[name + "_cv2"]).all(), name
    for name, src, mx, my in cases(with_cv2=False):          # the generator's inputs are these
        assert g[name + "_src"].tobytes() == src.tobytes() and g[name + "_mapx"].tobytes() == mx.tobytes(), name

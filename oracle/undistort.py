"""ORACLE SUPPORT (test infrastructure, NOT product code): a distorted pinhole camera as the reference's Frame handles it -
Frame::UndistortKeyPoints and Frame::ComputeImageBounds (src/Frame.cc:837-899), i.e. cv::undistortPoints(mvKeys, K, mDistCoef, noArray(), K)
restated in undistort_oracle.cpp - and the pieces of the RGB-D tests that use it: an RGB-D frame builder that also returns mvKeysUn, a
matcher FrameView with the undistorted image bounds, and oracle.chain.oracle_chain2 run with those bounds."""
import contextlib
import ctypes as C

import numpy as np

import oracle
from oracle import _p
from oracle import chain as _chain
from oracle import rgbd as _rgbd


def _camera(K):
    """(fx, fy, cx, cy) float32 from a 3x3 camera matrix or the four values."""
    K = np.asarray(K, np.float64)
    if K.shape == (3, 3):
        K = np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]])
    return np.ascontiguousarray(K.reshape(4), np.float32)


def undistort_points(xy, K, dist) -> np.ndarray:
    """cv::undistortPoints(src, dst, K, dist, noArray(), K) of float points (undistort_oracle.cpp) -> float32[n, 2]"""
    xy = np.ascontiguousarray(xy, np.float32).reshape(-1, 2)
    d = np.ascontiguousarray(dist, np.float32).reshape(-1)
    out = np.empty_like(xy)
    L = oracle.lib()
    L.orc_undistort_points.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    K = _camera(K)
    if L.orc_undistort_points(_p(xy), len(xy), _p(K), _p(d), len(d), _p(out)):
        raise ValueError(f"unsupported number of distortion coefficients: {len(d)}")
    return out


def image_bounds(W: int, H: int, K, dist) -> np.ndarray:
    """Frame::ComputeImageBounds (src/Frame.cc:871-899) -> float32 (mnMinX, mnMaxX, mnMinY, mnMaxY)"""
    d = np.ascontiguousarray(dist, np.float32).reshape(-1)
    out = np.empty(4, np.float32)
    L = oracle.lib()
    L.orc_image_bounds.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    K = _camera(K)
    if L.orc_image_bounds(W, H, _p(K), _p(d), len(d), _p(out)):
        raise ValueError(f"unsupported number of distortion coefficients: {len(d)}")
    return out


def undistort_keypoints(kps, K, dist) -> np.ndarray:
    """Frame::UndistortKeyPoints (src/Frame.cc:837-869): mvKeys when mDistCoef[0] == 0 (whatever the other coefficients are), else the
    keypoints with pt replaced by the undistorted points."""
    kps = np.ascontiguousarray(kps, oracle.KP_DTYPE)
    if np.float32(np.asarray(dist, np.float32).reshape(-1)[0]) == 0:
        return kps.copy()
    un = undistort_points(np.stack([kps["x"], kps["y"]], 1), K, dist)
    out = kps.copy()
    out["x"], out["y"] = un[:, 0], un[:, 1]
    return out


def rgbd_frame(extractor: "oracle.Extractor", gray: np.ndarray, depth_u16: np.ndarray, scale, bf: float, K, dist) -> dict:
    """The RGB-D Frame constructor (src/Frame.cc:200-237) of a camera with mDistCoef `dist`: ExtractORB, UndistortKeyPoints, then
    ComputeStereoFromRGBD on the scaled depth image - depth read at mvKeys, mvuRight from mvKeysUn.x
    -> dict(k = mvKeys, kun = mvKeysUn, d, depth, ur).  oracle_chain2 below takes frames with "k" = mvKeysUn (chain_frame)."""
    k, d, _ = extractor(gray)
    kun = undistort_keypoints(k, K, dist)
    dep, ur = oracle.depth_gather(_rgbd.depth_scale(depth_u16, scale), k, kun, bf)
    return dict(k=k, kun=kun, d=d, depth=dep, ur=ur)


def chain_frame(fr: dict) -> dict:
    """an rgbd_frame as the tracking chain sees it: the matchers, the edges and UnprojectStereo read mvKeysUn"""
    return dict(k=fr["kun"], d=fr["d"], depth=fr["depth"], ur=fr["ur"])


class FrameView(oracle.FrameView):
    """oracle.FrameView with the image bounds of ComputeImageBounds (mnMinX, mnMaxX, mnMinY, mnMaxY) instead of (0, W, 0, H)."""

    def __init__(self, *args, bounds):
        super().__init__(*args)
        self.c.min_x, self.c.max_x, self.c.min_y, self.c.max_y = (float(v) for v in bounds)


@contextlib.contextmanager
def _frame_bounds(bounds):
    """oracle.chain builds its frames with oracle.FrameView(...); within this block they get `bounds`."""
    plain = oracle.FrameView
    oracle.FrameView = lambda *args: FrameView(*args, bounds=bounds)
    try:
        yield
    finally:
        oracle.FrameView = plain


def oracle_chain2(frames, sf, pose0, W, H, cam, bounds, **kw):
    """oracle.chain.oracle_chain2 (same arguments and results) for frames of a distorted camera: `frames` carry mvKeysUn as "k"
    (chain_frame) and every Frame the chain's matchers see has the image bounds `bounds` (image_bounds)."""
    with _frame_bounds(bounds):
        return _chain.oracle_chain2(frames, sf, pose0, W, H, cam, **kw)

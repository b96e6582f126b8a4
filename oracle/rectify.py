"""ORACLE SUPPORT (test infrastructure, NOT product code): the stereo rectification System::TrackStereo runs when Settings::needToRectify()
(src/System.cc:251 ff.): cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of both images with the maps of cv::initUndistortRectifyMap, restated in
remap_oracle.cpp, and a stereo frame builder that rectifies a raw pair before the stereo Frame constructor (oracle/stereo.py)."""
import ctypes as C

import numpy as np

import oracle
from oracle import _p
from oracle import stereo as _stereo


def _lib():
    L = oracle.lib()
    vp, i = C.c_void_p, C.c_int
    L.orc_remap_u8.argtypes = [vp, i, i, i, vp, vp, i, i, i, vp, i]
    L.orc_convert_maps.argtypes = [vp, vp, i, i, i, vp, vp]
    return L


def remap(src: np.ndarray, mapx: np.ndarray, mapy: np.ndarray) -> np.ndarray:
    """cv2.remap(src, mapx, mapy, cv2.INTER_LINEAR) of a uint8 image with float32 maps (output of the maps' size)"""
    src = np.ascontiguousarray(src, np.uint8)
    mapx = np.ascontiguousarray(mapx, np.float32); mapy = np.ascontiguousarray(mapy, np.float32)
    assert mapx.shape == mapy.shape
    dh, dw = mapx.shape
    dst = np.empty((dh, dw), np.uint8)
    _lib().orc_remap_u8(_p(src), src.shape[1], src.shape[0], src.strides[0], _p(mapx), _p(mapy), dw, dw, dh, _p(dst), dw)
    return dst


def convert_maps(mapx: np.ndarray, mapy: np.ndarray):
    """cv2.convertMaps(mapx, mapy, cv2.CV_16SC2) -> (xy int16 [h, w, 2], a uint16 [h, w] = ay * 32 + ax)"""
    mapx = np.ascontiguousarray(mapx, np.float32); mapy = np.ascontiguousarray(mapy, np.float32)
    h, w = mapx.shape
    xy = np.empty((h, w, 2), np.int16); a = np.empty((h, w), np.uint16)
    _lib().orc_convert_maps(_p(mapx), _p(mapy), w, w, h, _p(xy), _p(a))
    return xy, a


def rectified_stereo_frame(ex_left: "oracle.Extractor", ex_right: "oracle.Extractor", left_raw: np.ndarray, right_raw: np.ndarray, maps, mb, mbf) -> dict:
    """System::TrackStereo with rectification: both raw images remapped (maps = (M1l, M2l, M1r, M2r)), then the stereo Frame constructor
    -> dict(k, d, depth, ur) as oracle.stereo.stereo_frame, plus the rectified images (left, right)."""
    m1l, m2l, m1r, m2r = maps
    left, right = remap(left_raw, m1l, m2l), remap(right_raw, m1r, m2r)
    fr = _stereo.stereo_frame(ex_left, ex_right, left, right, mb, mbf)
    fr["left"], fr["right"] = left, right
    return fr

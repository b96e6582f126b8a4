"""ORACLE SUPPORT (test infrastructure, NOT product code): the RGB-D input of System::TrackRGBD - Tracking::GrabImageRGBD
(src/Tracking.cc:1518) and the RGB-D Frame constructor (src/Frame.cc:200-237) - restated on the CPU for the tests of the RGB-D path:
the 16-bit depth PNG reader (png16_oracle.cpp), mDepthMapFactor, the 16U -> 32F scaling and an RGB-D frame builder whose output
oracle.chain.oracle_chain2 takes."""
import ctypes as C

import numpy as np

import oracle
from oracle import _p


def png_decode_depth16(png: bytes) -> np.ndarray:
    """cv::imread(IMREAD_UNCHANGED) of a 16-bit single-channel PNG stream (png16_oracle.cpp) -> uint16[h, w].  ValueError with the
    oracle's code for anything else (-2: not 16-bit gray non-interlaced)."""
    buf = np.frombuffer(png, np.uint8)
    w, h = C.c_int(0), C.c_int(0)
    L = oracle.lib()
    L.orc_png_decode_depth16.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    rc = L.orc_png_decode_depth16(_p(buf), len(buf), C.byref(w), C.byref(h), None, 0)
    if rc:
        raise ValueError(f"orc_png_decode_depth16: {rc}")
    out = np.empty((h.value, w.value), np.uint16)
    rc = L.orc_png_decode_depth16(_p(buf), len(buf), C.byref(w), C.byref(h), _p(out), out.size)
    if rc:
        raise ValueError(f"orc_png_decode_depth16: {rc}")
    return out


def depth_map_factor(factor: float) -> np.float32:
    """Tracking::mDepthMapFactor from RGBD.DepthMapFactor (src/Tracking.cc:1188-1204): 1.0f / factor in float, 1 when |factor| < 1e-5."""
    f = np.float32(factor)
    return np.float32(1.0) if abs(f) < np.float32(1e-5) else np.float32(np.float32(1.0) / f)


def depth_scale(u16: np.ndarray, scale) -> np.ndarray:
    """imDepth.convertTo(imDepth, CV_32F, mDepthMapFactor) of a CV_16U image (src/Tracking.cc:1538-1539): (float)u * (float)scale,
    rounded once per pixel."""
    return (np.asarray(u16, np.uint16).astype(np.float32) * np.float32(scale)).astype(np.float32)


def rgbd_frame(extractor: "oracle.Extractor", gray: np.ndarray, depth_u16: np.ndarray, scale, bf: float) -> dict:
    """The RGB-D Frame constructor (src/Frame.cc:200-237): ExtractORB, then ComputeStereoFromRGBD on the scaled depth image
    (mvKeysUn == mvKeys, k1 == 0) -> dict(k, d, depth, ur) as oracle.chain.oracle_chain2 takes it."""
    k, d, _ = extractor(gray)
    dep, ur = oracle.depth_gather(depth_scale(depth_u16, scale), k, k, bf)
    return dict(k=k, d=d, depth=dep, ur=ur)

"""ORACLE SUPPORT (test infrastructure): cv::resize(src, dst, size, 0, 0, INTER_LINEAR) of a CV_16UC1 image, System::TrackRGBD's resize of
the depth image when Settings::needToResize().  OpenCV's 16U linear resize runs in float32: per axis s = floor((d + 0.5) * scale - 0.5) with
the fraction f taken in double and rounded to float, weights 1 - f and f (s clamped to [0, n - 1] with f = 0, as for 8U), a horizontal
pass then a vertical pass, each a sum of two float products, then saturate_cast<ushort> (round half to even).  Pinned against cv2 at integer
factors (tests/test_oracle_resize.py); at other ratios OpenCV's sums differ in the last bits and the restatement is not claimed.  The 8-bit
resize is the pyramid's, oracle.resize_linear."""
import numpy as np


def _coefs(src_n: int, dst_n: int):
    fd = (np.arange(dst_n, dtype=np.float64) + 0.5) * (src_n / dst_n) - 0.5
    s = np.floor(fd).astype(np.int64)
    f = (fd - s).astype(np.float32)
    clamp = (s < 0) | (s >= src_n - 1)
    s = np.clip(s, 0, src_n - 1)
    f[clamp] = 0
    return s, np.minimum(s + 1, src_n - 1), (np.float32(1) - f).astype(np.float32), f


def resize_linear_u16(src: np.ndarray, dw: int, dh: int) -> np.ndarray:
    """cv2.resize(src, (dw, dh), interpolation=cv2.INTER_LINEAR) of a uint16 image (float32 arithmetic, one rounding per operation)"""
    src = np.asarray(src, np.uint16)
    sx0, sx1, a0, a1 = _coefs(src.shape[1], dw)
    sy0, sy1, b0, b1 = _coefs(src.shape[0], dh)
    img = src.astype(np.float32)
    row = (img[:, sx0] * a0).astype(np.float32) + (img[:, sx1] * a1).astype(np.float32)
    out = (row[sy0] * b0[:, None]).astype(np.float32) + (row[sy1] * b1[:, None]).astype(np.float32)
    return np.clip(np.rint(out), 0, 65535).astype(np.uint16)


def resize_linear(src: np.ndarray, dw: int, dh: int) -> np.ndarray:
    """the oracle's cv2.resize(INTER_LINEAR) of a uint8 (oracle.resize_linear) or uint16 image"""
    import oracle
    return oracle.resize_linear(src, dw, dh) if src.dtype == np.uint8 else resize_linear_u16(src, dw, dh)

"""The RGB-D input oracle (System::TrackRGBD's GrabImageRGBD): the 16-bit depth PNG decoder (oracle/png16_oracle.cpp) against
python-cv2's imdecode(IMREAD_UNCHANGED), live and through tests/golden/png16_golden.npz, and oracle.rgbd.depth_scale against OpenCV's
scaled 16U -> 32F conversion for every uint16 value, live and through SHA-256 digests of cv2's outputs."""
import hashlib
import struct
import zlib
from pathlib import Path

import numpy as np
import pytest

from oracle import rgbd as R
from orb_slam3_rgbl_b200 import synthetic as S

GOLD = Path(__file__).resolve().parent / "golden" / "png16_golden.npz"
FACTORS = (1, 256, 1000, 5000)
# sha256 of cv2.multiply(u, float(np.float32(1) / np.float32(f)), dtype=cv2.CV_32F).tobytes() for u = arange(65536).reshape(256, 256) as
# uint16 (python-cv2 4.13.0); cv2 does not expose Mat::convertTo, and this scaled multiply is the same per-pixel rule d = (float)u * alpha
CV2_SCALE_SHA256 = {
    1: "00f2c484030d0c6a5f5a383847c4d056c56aa4de87977cd995dc311f97909a7f",
    256: "56033a8c262b423706f646d67b7badaac3ca8ae70037d831284e0a374cd59b48",
    1000: "0ebf05dba01f3f170772c59d08d0426aa9b5a5daf03a79c6c83a6d3538a97fed",
    5000: "14e1286d0f196eae538a3f3fc616d79266f9f1c353bcb2ec3a56d4d855824197",
}


def cases():
    """(name, png bytes): all five filters cycling row by row, random filters per row, several IDAT chunk sizes, a KITTI-like depth image."""
    rng = np.random.default_rng(16)
    u = rng.integers(0, 65536, (61, 47)).astype(np.uint16)
    seq = S.PlaneSequence(5, 2, W=333, H=140)
    d = seq.depth16(1, 256.0, 0.1)
    out = [("cycle", S.encode_png16(u)), ("random", S.encode_png16(u, rng.integers(0, 5, len(u)))),
           ("chunk7", S.encode_png16(u, None, 7)), ("chunk1000", S.encode_png16(u, rng.integers(0, 5, len(u)), 1000)),
           ("plane", S.encode_png16(d, None, 4096))]
    for ft in range(5):
        out.append((f"filter{ft}", S.encode_png16(u, np.full(len(u), ft))))
    return out


def cv2_reference(png: bytes) -> np.ndarray:
    import cv2
    m = cv2.imdecode(np.frombuffer(png, np.uint8), cv2.IMREAD_UNCHANGED)
    assert m.dtype == np.uint16 and m.ndim == 2
    return m


def test_depth16_decoder_matches_cv2_live():
    pytest.importorskip("cv2")
    for name, png in cases():
        assert (R.png_decode_depth16(png) == cv2_reference(png)).all(), name


def test_depth16_decoder_matches_golden():
    g = np.load(GOLD)
    for name, png in cases():
        assert (g[name + "_png"].tobytes() == png), name          # the generator still makes the committed streams
        assert (R.png_decode_depth16(png) == g[name + "_depth"]).all(), name


def _with_ihdr(png: bytes, **fields) -> bytes:
    """the stream with IHDR bytes replaced (bit depth 8, colour type 9, interlace 12) and the chunk CRC recomputed"""
    b = bytearray(png)
    for off, v in fields.values():
        b[16 + off] = v
    b[29:33] = struct.pack(">I", zlib.crc32(bytes(b[12:29])) & 0xffffffff)
    return bytes(b)


def rejected_depth_streams():
    u = np.random.default_rng(3).integers(0, 65536, (20, 30)).astype(np.uint16)
    return [("8-bit", S.encode_png(u.astype(np.uint8))), ("16-bit RGB", S.encode_png16(np.stack([u, u, u], -1))),
            ("interlaced", _with_ihdr(S.encode_png16(u), interlace=(12, 1)))]


def test_depth16_decoder_rejects_other_formats():
    for name, png in rejected_depth_streams():
        with pytest.raises(ValueError, match="-2"):
            R.png_decode_depth16(png)


def test_depth_scale_matches_cv2_live():
    cv2 = pytest.importorskip("cv2")
    u = np.arange(65536, dtype=np.uint16).reshape(256, 256)
    for f in FACTORS:
        s = R.depth_map_factor(f)
        ref = cv2.multiply(u, float(s), dtype=cv2.CV_32F)
        assert (R.depth_scale(u, s).view(np.uint32) == ref.view(np.uint32)).all(), f


def test_depth_scale_matches_cv2_digests():
    u = np.arange(65536, dtype=np.uint16).reshape(256, 256)
    for f in FACTORS:
        got = R.depth_scale(u, R.depth_map_factor(f))
        assert hashlib.sha256(np.ascontiguousarray(got).tobytes()).hexdigest() == CV2_SCALE_SHA256[f], f


def test_depth_map_factor_rule():
    """mDepthMapFactor = 1.0f / RGBD.DepthMapFactor in float, and 1 for |factor| < 1e-5 (src/Tracking.cc:1188-1204)"""
    assert R.depth_map_factor(5000) == np.float32(1) / np.float32(5000)
    assert R.depth_map_factor(0.0) == 1.0 and R.depth_map_factor(5e-6) == 1.0

"""The CPU side of stereo rectification: the synthetic rig's rectification maps against cv2.initUndistortRectifyMap, its raw views, and
the oracle's tracking chain on oracle-rectified raw pairs of a distorted stereo sequence against the synthetic truth (and against the same
raw images tracked as if they were rectified)."""
import numpy as np
import pytest

import oracle
from oracle import chain as CH
from oracle import rectify as RC
from oracle import stereo as ST
from orb_slam3_rgbl_b200 import synthetic as S

CAM = S.EUROC_CAM
W, H = S.EUROC_W, S.EUROC_H
MB = float(np.float32(CAM[4]) / np.float32(CAM[0]))
MBF = float(CAM[4])
# Accuracy bounds of the rectified distorted sequence (15 frames), fixed from the CPU run of test_oracle_chain_on_rectified_pairs and used by
# tests/test_gpu_rectify.py too.  Oracle, K = 2 / K = 0: x 0.090 / 0.072, y 0.060 / 0.065, z 0.015 / 0.007 m; median |mvDepth - Z| 0.35 m.
# The same raw images tracked as if they were rectified: z 0.061 / 0.037 m, median depth error 4.5 m.  (A pinhole sequence of this camera
# tracks to x 0.041, y 0.013, z 0.005 m over 11 frames: most of the x / y error is this camera's, not the rectification's.)
RECTIFIED_MAX_XY_ERR, RECTIFIED_MAX_Z_ERR, RECTIFIED_MAX_DEPTH_ERR = 0.12, 0.025, 0.6
RAW_MIN_Z_ERR, RAW_MIN_DEPTH_ERR = 0.03, 2.0


def errors(seq, poses, frames):
    """max |error| of the camera centre along x, y, z over the frames, and the median |mvDepth - Z| of the stereo matches"""
    truth = np.array([seq.pose(t) for t in range(len(poses))])
    e = np.abs(np.asarray(poses)[:, 4:7] - truth[:, 4:7]).max(0)
    d = np.concatenate([f["depth"][f["depth"] > 0] for f in frames])
    return e, float(np.median(np.abs(d - seq.Z)))


def rig_rotations():
    """a small rotation of the left and of the right camera (R1, R2 of a stereoRectify-like rig with R != I)"""
    def rot(rx, ry, rz):
        a = np.array([rx, ry, rz]); t = np.linalg.norm(a); k = a / t
        Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
        return np.eye(3) + np.sin(t) * Kx + (1 - np.cos(t)) * Kx @ Kx
    return rot(0.012, -0.02, 0.004), rot(-0.008, 0.015, -0.006)


def sequence(seed=51, n=16):
    return S.PlaneSequence(seed, n, W=W, H=H, cam=CAM, dist=S.EUROC_DIST)


def test_rectification_maps_match_cv2():
    cv2 = pytest.importorskip("cv2")
    seq = sequence(n=2)
    fx, fy, cx, cy = CAM[:4]
    K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]])
    for R in (None,) + rig_rotations():
        mx, my = seq.rectification_maps(R)
        cx_, cy_ = cv2.initUndistortRectifyMap(K, S.EUROC_DIST, np.eye(3) if R is None else R, K, (W, H), cv2.CV_32FC1)
        assert mx.dtype == np.float32 and mx.shape == (H, W)
        assert np.abs(mx - cx_).max() < 1e-3 and np.abs(my - cy_).max() < 1e-3


def test_raw_views():
    """the raw left view is image(t); rectifying the raw pair gives the pinhole views (up to the two resamplings); image(t), right_image
    and disparity_px keep refusing a distorted sequence"""
    seq = sequence(n=4)
    assert seq.raw_left_image(2).tobytes() == seq.image(2).tobytes()
    with pytest.raises(ValueError):
        seq.right_image(0)
    mx, my = seq.rectification_maps()
    m, s = seq.margin, seq.step_index(2)
    for img, d in ((seq.raw_left_image(2), 0), (seq.raw_right_image(2), 5)):
        pin = seq.texture[m:m + H, s * seq.shift + d + m:s * seq.shift + d + m + W].astype(np.int64)
        assert np.abs(RC.remap(img, mx, my).astype(np.int64) - pin).mean() < 4.0
        assert np.abs(img.astype(np.int64) - pin).mean() > 20.0
    with pytest.raises(ValueError):
        S.PlaneSequence(1, 2).raw_right_image(0)


def oracle_poses(seq, frames, K=2):
    sf = oracle.Extractor(2000).scale_factors.copy()
    poses, *_ = CH.oracle_chain2(frames, sf, seq.pose(0), W, H, CAM, K=K, th_last=7.0, th_local=1.0)
    return np.asarray(poses)


def test_oracle_chain_on_rectified_pairs():
    """oracle_chain2 on the oracle's rectified stereo frames of the distorted sequence stays within the bounds above; the same raw images
    tracked as if they were rectified have a clearly larger error along the depth axis and far worse stereo depths"""
    seq = sequence()
    n = 15
    maps = seq.rectification_maps() * 2
    exl, exr = oracle.Extractor(2000), oracle.Extractor(2000)
    rect = [RC.rectified_stereo_frame(exl, exr, seq.raw_left_image(t), seq.raw_right_image(t), maps, MB, MBF) for t in range(n)]
    raw = [ST.stereo_frame(exl, exr, seq.raw_left_image(t), seq.raw_right_image(t), MB, MBF) for t in range(n)]
    assert (np.array([(f["depth"] > 0).sum() for f in rect]) > 300).all()
    for K in (2, 0):
        e, dep = errors(seq, oracle_poses(seq, rect, K), rect)
        assert e[0] < RECTIFIED_MAX_XY_ERR and e[1] < RECTIFIED_MAX_XY_ERR and e[2] < RECTIFIED_MAX_Z_ERR and dep < RECTIFIED_MAX_DEPTH_ERR, (K, e, dep)
        e, dep = errors(seq, oracle_poses(seq, raw, K), raw)
        assert e[2] > RAW_MIN_Z_ERR and dep > RAW_MIN_DEPTH_ERR, (K, e, dep)

"""The undistortion oracle (oracle/undistort_oracle.cpp: cv::undistortPoints as Frame::UndistortKeyPoints and Frame::ComputeImageBounds
call it) against python-cv2, live and through tests/golden/undistort_golden.npz: points in and around a 640 x 480 image, its corners, far
points that take OpenCV's icdist < 0 branch, 4- and 5-coefficient sets; the reference's k1 == 0 early return."""
from pathlib import Path

import numpy as np
import pytest

import oracle
import oracle.chain  # noqa: F401
from oracle import undistort as U
from orb_slam3_rgbl_b200 import synthetic as S

GOLD = Path(__file__).resolve().parent / "golden" / "undistort_golden.npz"
CAM = (S.TUM1_FX, S.TUM1_FY, S.TUM1_CX, S.TUM1_CY)
W, H = S.TUM_W, S.TUM_H


def sets():
    """(name, dist): TUM1's five coefficients and its first four, a barrel lens, and k1 == 0 with the other coefficients non-zero"""
    return [("tum1", S.TUM1_DIST), ("tum1_4", S.TUM1_DIST[:4].copy()), ("barrel", np.array([-0.31, 0.11, 0.0012, -0.0021, -0.02], np.float32)),
            ("k1zero", np.array([0.0, -0.95, 0.004, 0.002, 1.1], np.float32))]


def points(name, n):
    """seeded points over the image and a 20 px margin, its four corners, and (tum1_4) points far outside it"""
    rng = np.random.default_rng(len(name) * 7919 + n)
    xy = np.stack([rng.uniform(-20, W + 20, n), rng.uniform(-20, H + 20, n)], 1)
    corners = [[0, 0], [W, 0], [0, H], [W, H]]
    far = np.stack([rng.uniform(-3000, W + 3000, n // 4), rng.uniform(-3000, H + 3000, n // 4)], 1) if name == "tum1_4" else np.zeros((0, 2))
    return np.ascontiguousarray(np.concatenate([corners, xy, far]), np.float32)


def camera_matrix():
    return np.array([[CAM[0], 0, CAM[2]], [0, CAM[1], CAM[3]], [0, 0, 1]], np.float32)


def cv2_undistort(xy, dist):
    import cv2
    return cv2.undistortPoints(xy.reshape(-1, 1, 2), camera_matrix(), dist, None, camera_matrix()).reshape(-1, 2)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def test_icdist_branch_is_covered():
    """the far points of tum1_4 include points whose first icdist is negative (OpenCV then returns the distorted point's normalised
    coordinates), and they are not rare"""
    k1, k2 = (float(v) for v in S.TUM1_DIST[:2])
    xy = points("tum1_4", 4000).astype(np.float64)
    x, y = (xy[:, 0] - CAM[2]) / CAM[0], (xy[:, 1] - CAM[3]) / CAM[1]
    r2 = x * x + y * y
    assert ((1 + (k2 * r2 + k1) * r2) < 0).sum() > 100


def test_undistort_matches_cv2_live():
    pytest.importorskip("cv2")
    for name, dist in sets():
        xy = points(name, 50000)
        assert (_bits(U.undistort_points(xy, CAM, dist)) == _bits(cv2_undistort(xy, dist))).all(), name


def test_undistort_matches_golden():
    g = np.load(GOLD)
    for name, dist in sets():
        xy = points(name, 4000)
        assert (g[name + "_xy"].tobytes() == xy.tobytes()) and (g[name + "_dist"].tobytes() == dist.tobytes()), name    # same inputs
        assert (_bits(U.undistort_points(xy, CAM, dist)) == _bits(g[name + "_cv2"])).all(), name


def _cv2_bounds(undist_corners):
    c = undist_corners
    return np.array([min(c[0, 0], c[2, 0]), max(c[1, 0], c[3, 0]), min(c[0, 1], c[1, 1]), max(c[2, 1], c[3, 1])], np.float32)


def test_image_bounds_match_cv2_corners():
    """ComputeImageBounds (src/Frame.cc:871-899) from cv2's undistorted corners (live, else the golden file's first four points)"""
    try:
        import cv2  # noqa: F401
        live = True
    except ImportError:
        live = False
    g = np.load(GOLD)
    for name, dist in sets():
        corners = cv2_undistort(points(name, 4000)[:4], dist) if live else g[name + "_cv2"][:4]
        b = U.image_bounds(W, H, CAM, dist)
        if dist[0] == 0:
            assert list(b) == [0, W, 0, H], name                       # the reference's else branch, whatever k2..k3 are
        else:
            assert b.tobytes() == _cv2_bounds(corners).tobytes(), name


def test_k1_zero_is_the_identity():
    """Frame::UndistortKeyPoints returns mvKeysUn = mvKeys when mDistCoef[0] == 0, even with k2, p1, p2, k3 != 0 (src/Frame.cc:837-843),
    although cv::undistortPoints would move the points"""
    dist = dict(sets())["k1zero"]
    k = np.zeros(500, oracle.KP_DTYPE)
    xy = points("k1zero", 496)
    k["x"], k["y"], k["octave"], k["angle"] = xy[:, 0], xy[:, 1], 3, 17.5
    assert U.undistort_keypoints(k, CAM, dist).tobytes() == k.tobytes()
    assert (_bits(U.undistort_points(xy, CAM, dist)) != _bits(xy)).any()
    kun = U.undistort_keypoints(k, CAM, S.TUM1_DIST)
    for f in ("size", "angle", "response", "octave", "class_id"):
        assert (kun[f] == k[f]).all(), f                               # only pt changes


def test_chain_with_bounds_tracks_the_distorted_sequence():
    """U.oracle_chain2 gives every Frame of the chain the undistorted image bounds (and leaves oracle.FrameView as it was); on mvKeysUn
    frames of the distorted synthetic sequence it stays within 1 cm of the truth, which the distorted keypoints do not"""
    cam = CAM + (S.TUM1_BF,)
    seq = S.PlaneSequence(56, 6, Z=3.0, W=W, H=H, cam=cam, dist=S.TUM1_DIST)
    ex = oracle.Extractor(1000)
    scale = np.float32(1.0) / np.float32(S.TUM_DEPTH_FACTOR)
    frames = [U.rgbd_frame(ex, seq.image(t), seq.depth16(t, S.TUM_DEPTH_FACTOR, 0.05), scale, S.TUM1_BF, CAM, S.TUM1_DIST) for t in range(6)]
    bounds = U.image_bounds(W, H, CAM, S.TUM1_DIST)
    fv = U.FrameView(frames[0]["kun"], frames[0]["ur"], frames[0]["d"], W, H, ex.scale_factors, *cam, bounds=bounds)
    assert (fv.c.min_x, fv.c.max_x, fv.c.min_y, fv.c.max_y) == tuple(float(v) for v in bounds)
    plain = oracle.FrameView
    truth = np.array([seq.pose(t)[4] for t in range(6)])
    poses = U.oracle_chain2([U.chain_frame(f) for f in frames], ex.scale_factors.copy(), seq.pose(0), W, H, cam, bounds, K=2)[0]
    assert oracle.FrameView is plain
    assert np.abs(poses[:, 4] - truth).max() < 0.01
    raw = oracle.chain.oracle_chain2([dict(k=f["k"], d=f["d"], depth=f["depth"], ur=f["ur"]) for f in frames], ex.scale_factors.copy(),
                                     seq.pose(0), W, H, cam, K=2)[0]
    assert np.abs(raw[:, 4] - truth).max() > np.abs(poses[:, 4] - truth).max()

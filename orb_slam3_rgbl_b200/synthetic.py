"""Seeded synthetic KITTI-like inputs (SURVEY.md §8(d)); KITTI itself is not available offline.

Everything is numpy-only and deterministic given the seed, so the CPU box and the GPU box
generate identical bytes.  Formats follow the reference's example driver:
  * image: uint8 gray H x W (``cv::imread`` + cvtColor, src/Tracking.cc:1567-1580)
  * point cloud: float32 4 x N planar rows (x, y, z, 1) (Examples/RGB-L/rgbl_kitti.cc:168-177)
  * calibration: Examples/RGB-L/KITTI00-02.yaml
"""
from __future__ import annotations

import numpy as np

# Examples/RGB-L/KITTI00-02.yaml:9-12,29,44-55,63-64
KITTI_FX = 718.856
KITTI_FY = 718.856
KITTI_CX = 607.1928
KITTI_CY = 185.2157
KITTI_BF = 100.0
KITTI_W, KITTI_H = 1241, 376
KITTI_TR = np.array([[4.276802385584e-04, -9.999672484946e-01, -8.084491683471e-03, -1.198459927713e-02],
                     [-7.210626507497e-03, 8.081198471645e-03, -9.999413164504e-01, -5.403984729748e-02],
                     [9.999738645903e-01, 4.859485810390e-04, -7.206933692422e-03, -2.921968648686e-01]], np.float64)
LIDAR_MIN_DIST, LIDAR_MAX_DIST = 5.0, 200.0
# ORB-SLAM3's Examples/RGB-D/TUM1.yaml (TUM RGB-D fr1 sequences): a 640 x 480 camera with non-zero distortion
TUM_W, TUM_H = 640, 480
TUM1_FX, TUM1_FY, TUM1_CX, TUM1_CY = 517.306408, 516.469215, 318.643040, 255.313989
TUM1_DIST = np.array([0.262383, -0.953104, -0.005358, 0.002628, 1.163314], np.float32)      # k1, k2, p1, p2, k3
TUM1_BF = 40.0
TUM_DEPTH_FACTOR = 5000.0
# a EuRoC-like stereo camera (752 x 480, strong barrel distortion) for the rectification path; bf is chosen so that the plane sequences
# (Z = 20 m) have a whole-pixel disparity of 5 px, not EuRoC's own baseline
EUROC_W, EUROC_H = 752, 480
EUROC_CAM = (458.654, 457.296, 367.215, 248.375, 100.0)          # fx, fy, cx, cy, bf
EUROC_DIST = np.array([-0.28, 0.07, 2e-4, 2e-5], np.float32)      # k1, k2, p1, p2


def camera_matrix(fx=KITTI_FX, fy=KITTI_FY, cx=KITTI_CX, cy=KITTI_CY) -> np.ndarray:
    return np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)


def lidar_projection_matrix(K: np.ndarray | None = None, Tr: np.ndarray | None = None) -> np.ndarray:
    """3x4 float32 P = K[3x3|0] * [Tr;0001] (src/DepthModule.cc:434 builds it once on the host).

    NOTE: the reference's product is evaluated by OpenCV's small-matrix path; callers that need the
    reference's exact 12 floats must pass them across the ABI.  Here (synthetic calibration) the
    float32(float64 product) is the definition.
    """
    K = camera_matrix() if K is None else K
    Tr = KITTI_TR if Tr is None else Tr
    return (K.astype(np.float64) @ Tr.astype(np.float64)).astype(np.float32)


def _upsample_bilinear(a: np.ndarray, H: int, W: int) -> np.ndarray:
    h, w = a.shape
    ys = np.linspace(0, h - 1, H); xs = np.linspace(0, w - 1, W)
    y0 = np.floor(ys).astype(int); x0 = np.floor(xs).astype(int)
    y1 = np.minimum(y0 + 1, h - 1); x1 = np.minimum(x0 + 1, w - 1)
    fy = (ys - y0)[:, None]; fx = (xs - x0)[None, :]
    top = a[y0][:, x0] * (1 - fx) + a[y0][:, x1] * fx
    bot = a[y1][:, x0] * (1 - fx) + a[y1][:, x1] * fx
    return top * (1 - fy) + bot * fy


def make_image(seed: int, W: int = KITTI_W, H: int = KITTI_H, n_rects: int = 350) -> np.ndarray:
    """Multi-octave value noise plus random rectangles (real corners); ~10-20k FAST candidates at 1241x376."""
    rng = np.random.default_rng(seed)
    img = np.zeros((H, W), np.float64)
    for div, amp in ((32, 70.0), (8, 35.0), (2, 10.0)):
        h, w = max(2, H // div + 2), max(2, W // div + 2)
        img += amp * _upsample_bilinear(rng.random((h, w)), H, W)
    img += 40.0
    scale = np.sqrt(W * H / float(KITTI_W * KITTI_H))
    for _ in range(int(n_rects * scale * scale)):
        rw = int(rng.integers(6, 70)); rh = int(rng.integers(6, 50))
        x = int(rng.integers(0, W - 1)); y = int(rng.integers(0, H - 1))
        delta = float(rng.integers(25, 90)) * (1 if rng.random() < 0.5 else -1)
        img[y:y + rh, x:x + rw] += delta
    img += rng.normal(0.0, 1.5, (H, W))
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def make_pointcloud(seed: int, n_rings: int = 64, n_azimuth: int = 1875, W: int = KITTI_W, H: int = KITTI_H) -> np.ndarray:
    """Velodyne-like sweep, ring-major azimuth order, float32 4 x N planar (x, y, z, 1).

    Range comes from a ground plane (sensor 1.73 m above ground) plus random boxes (5-80 m), 2 cm noise.
    Roughly 15-20 % of the points land in a KITTI image.
    """
    rng = np.random.default_rng(seed ^ 0x5EED)
    elev = np.deg2rad(np.linspace(2.0, -24.8, n_rings))[:, None]
    azim = np.linspace(-np.pi, np.pi, n_azimuth, endpoint=False)[None, :]
    ce, se = np.cos(elev), np.sin(elev)
    # ground plane range
    with np.errstate(divide="ignore"):
        r_ground = np.where(se < -1e-3, 1.73 / -se, 120.0)
    r = np.minimum(r_ground, 120.0) * np.ones_like(azim)
    # random "boxes": azimuth sectors at closer range
    for _ in range(40):
        a0 = rng.uniform(-np.pi, np.pi); aw = rng.uniform(0.03, 0.35)
        dist = rng.uniform(5.0, 80.0)
        top = rng.uniform(-0.02, 0.04)
        sel = (np.abs(((azim - a0 + np.pi) % (2 * np.pi)) - np.pi) < aw)
        hit = sel & (elev < top) & (r * ce > dist)
        r = np.where(hit, dist / np.maximum(ce, 1e-3), r)
    r = r + rng.normal(0.0, 0.02, r.shape)
    x = (r * ce * np.cos(azim)).ravel(); y = (r * ce * np.sin(azim)).ravel(); z = (r * se).ravel()
    pts = np.stack([x, y, z, np.ones_like(x)]).astype(np.float32)
    return np.ascontiguousarray(pts)


def make_frame(seed: int, W: int = KITTI_W, H: int = KITTI_H, n_azimuth: int = 1875):
    return make_image(seed, W, H), make_pointcloud(seed, 64, n_azimuth, W, H)


def structuring_element(kind: str, ku: int, kv: int | None = None) -> np.ndarray:
    """0/1 uint8 mask [kv, ku] for DepthModule::Upsample_InverseDilation (src/DepthModule.cc:234-260).

    'Diamond' follows include/DepthModule.h:138-161 (|dx|+|dy| <= r); 'Rectangle'/'Cross'/'Ellipse'
    follow cv::getStructuringElement.
    """
    kv = ku if kv is None else kv
    kind = kind.lower()
    m = np.zeros((kv, ku), np.uint8)
    if kind == "rectangle":
        m[:] = 1
    elif kind == "cross":
        m[kv // 2, :] = 1; m[:, ku // 2] = 1
    elif kind == "diamond":
        if ku not in (3, 5, 7, 9):
            raise ValueError("invalid kernel size for diamond kernel")   # DepthModule.cc:250-253
        r = ku // 2
        m = np.zeros((ku, ku), np.uint8)
        for j in range(ku):
            for i in range(ku):
                m[j, i] = 1 if abs(i - r) + abs(j - r) <= r else 0
    elif kind == "ellipse":
        r, c = kv // 2, ku // 2
        inv_r2 = 1.0 / (r * r) if r else 0.0
        for i in range(kv):
            dy = i - r
            if abs(dy) <= r:
                dx = int(np.rint(c * np.sqrt((r * r - dy * dy) * inv_r2)))
                m[i, max(c - dx, 0):min(c + dx + 1, ku)] = 1
    else:
        raise ValueError(f"invalid kernel type: {kind}")
    return m


# ------------------------------------------------------------------------------------------------
# A geometrically consistent synthetic sequence (SURVEY.md 8(d) "Sequence"): a textured fronto-parallel
# plane at depth Z seen by a camera translating along +x.  Frame t is an integer-pixel crop of one big
# texture, so consecutive frames show the same corners shifted by `shift_px`; the LiDAR points are the
# ring/azimuth rays intersected with the same plane, expressed in the Velodyne frame of each pose.
# ------------------------------------------------------------------------------------------------

class PlaneSequence:
    """Camera translating along +x in front of a textured plane at depth Z (image shift shift_px per frame) with a Velodyne-like fan of
    points on the plane.  loop > 0: the camera turns round after loop / 2 frames and is back at the start after `loop` frames, so that a
    sequence of any length stays on the texture and consecutive passes over the same `loop` frames form one continuous trajectory."""

    def __init__(self, seed: int, n_frames: int, shift_px: int = 7, Z: float = 20.0, W: int = KITTI_W, H: int = KITTI_H,
                 n_rings: int = 64, n_azimuth: int = 1875, loop: int = 0, cam=None, dist=None):
        """dist: the camera's distortion (k1, k2, p1, p2[, k3], OpenCV's model); image(t) is then the distorted view of the scene."""
        self.seed, self.n_frames, self.shift, self.Z, self.W, self.H = seed, n_frames, shift_px, Z, W, H
        self.cam = tuple(cam) if cam is not None else (KITTI_FX, KITTI_FY, KITTI_CX, KITTI_CY, KITTI_BF)      # (fx, fy, cx, cy, bf)
        self.loop = loop
        span = (loop // 2 + 1) if loop > 0 else n_frames
        self.dist = None if dist is None else np.asarray(dist, np.float64).reshape(-1)
        if self.dist is None:
            self.texture = make_image(seed, W + shift_px * span + 8, H)
        else:
            # where each pixel of the distorted image sees the undistorted (pinhole) image, and a texture margin that covers it
            self.map_x, self.map_y = undistorted_pixel_map(W, H, self.cam[:4], self.dist)
            self.margin = int(np.ceil(max(-self.map_x.min(), -self.map_y.min(), self.map_x.max() - (W - 1), self.map_y.max() - (H - 1), 0.0))) + 2
            m = self.margin
            self.texture = make_image(seed, W + shift_px * span + 8 + 2 * m, H + 2 * m)
        self.dX = shift_px * Z / self.cam[0]         # camera translation per frame (metres along +x)
        self.n_rings, self.n_az = n_rings, n_azimuth
        Tr4 = np.eye(4); Tr4[:3] = KITTI_TR
        self.Tr_inv = np.linalg.inv(Tr4)
        self.P = lidar_projection_matrix(camera_matrix(*self.cam[:4]))

    def step_index(self, t: int) -> int:
        """Position of frame t on the track, in steps of dX (triangle wave when the sequence loops)."""
        if self.loop <= 0:
            return t
        r = t % self.loop
        return r if r <= self.loop // 2 else self.loop - r

    def image(self, t: int) -> np.ndarray:
        s = self.step_index(t)
        if self.dist is None:
            return np.ascontiguousarray(self.texture[:, s * self.shift: s * self.shift + self.W])
        # the pinhole view of frame t is the texture crop at (s * shift + margin, margin); sample it bilinearly where the lens maps each pixel
        tex = self.texture.astype(np.float64)
        xs = self.map_x + (s * self.shift + self.margin); ys = self.map_y + self.margin
        x0 = np.floor(xs).astype(np.int64); y0 = np.floor(ys).astype(np.int64)
        fx = xs - x0; fy = ys - y0
        top = tex[y0, x0] * (1 - fx) + tex[y0, x0 + 1] * fx
        bot = tex[y0 + 1, x0] * (1 - fx) + tex[y0 + 1, x0 + 1] * fx
        return np.ascontiguousarray(np.clip(np.rint(top * (1 - fy) + bot * fy), 0, 255).astype(np.uint8))

    def raw_left_image(self, t: int) -> np.ndarray:
        """Frame t of the left camera of a distorted stereo rig (a sequence built with dist=), before rectification: image(t)."""
        if self.dist is None:
            raise ValueError("raw_left_image needs a sequence with a distortion model (dist=)")
        return self.image(t)

    def raw_right_image(self, t: int) -> np.ndarray:
        """Frame t of the right camera of a distorted stereo rig (same lens, baseline bf / fx along +x, no rotation), before rectification:
        the lens sampling of image(t) applied to the pinhole view shifted by the disparity d = bf / Z (right_image of a pinhole sequence).
        Rectified with rectification_maps(), it becomes that pinhole view."""
        if self.dist is None:
            raise ValueError("raw_right_image needs a sequence with a distortion model (dist=)")
        s, d = self.step_index(t), self._whole_disparity()
        tex = self.texture.astype(np.float64)
        xs = self.map_x + (s * self.shift + d + self.margin); ys = self.map_y + self.margin
        x0 = np.floor(xs).astype(np.int64); y0 = np.floor(ys).astype(np.int64)
        fx = xs - x0; fy = ys - y0
        top = tex[y0, x0] * (1 - fx) + tex[y0, x0 + 1] * fx
        bot = tex[y0 + 1, x0] * (1 - fx) + tex[y0 + 1, x0 + 1] * fx
        return np.ascontiguousarray(np.clip(np.rint(top * (1 - fy) + bot * fy), 0, 255).astype(np.uint8))

    def rectification_maps(self, R=None):
        """float32 (map_x, map_y), H x W, of cv::initUndistortRectifyMap(K, dist, R, K, (W, H), CV_32FC1) for this sequence's camera, in
        closed form: rectified pixel (u, v) -> ray R^-1 K^-1 (u, v, 1) -> distort_normalized -> K.  R = None: the identity (the maps of the
        raw views above, whose rig needs no rotation)."""
        if self.dist is None:
            raise ValueError("rectification_maps needs a sequence with a distortion model (dist=)")
        return rectification_maps(self.W, self.H, self.cam[:4], self.dist, R)

    def disparity_px(self) -> int:
        """Disparity of the plane in a rectified stereo rig with baseline bf / fx: bf / Z pixels (5 at the defaults)."""
        if self.dist is not None:
            raise ValueError("right_image needs a pinhole camera: stereo pairs are rectified, this sequence has a distortion model")
        return self._whole_disparity()

    def _whole_disparity(self) -> int:
        d = self.cam[4] / self.Z
        if abs(d - round(d)) > 1e-9:
            raise ValueError(f"right_image needs a whole-pixel disparity bf / Z, got {d} px")
        if round(d) > self.shift + 8:
            raise ValueError(f"disparity {d} px exceeds the texture's slack of shift_px + 8 = {self.shift + 8} px beyond the last crop")
        return int(round(d))

    def right_image(self, t: int) -> np.ndarray:
        """Frame t of the right camera of a rectified stereo rig (baseline bf / fx along +x): the plane point at left pixel u appears at
        u - d, d = bf / Z, so the view is the texture crop of image(t) shifted by d columns."""
        s, d = self.step_index(t), self.disparity_px()
        return np.ascontiguousarray(self.texture[:, s * self.shift + d: s * self.shift + d + self.W])

    def pose(self, t: int) -> np.ndarray:
        """Tcw as (qx, qy, qz, qw, tx, ty, tz): identity rotation, camera centre at x = step_index(t) * dX."""
        return np.array([0, 0, 0, 1, -self.step_index(t) * self.dX, 0, 0], np.float32)

    def depth16(self, t: int, factor: float = 256.0, hole_frac: float = 0.05, noise_m: float = 0.01) -> np.ndarray:
        """uint16 H x W depth image of frame t as an RGB-D sensor delivers it (CV_16U, metres x factor; KITTI depth PNGs use 256, TUM
        5000): the plane's depth Z with seeded Gaussian noise, rounded, and a seeded fraction of holes (0 = no measurement)."""
        rng = np.random.default_rng(self.seed * 104729 + t)
        d = self.Z + rng.normal(0.0, noise_m, (self.H, self.W))
        u = np.clip(np.rint(d * factor), 0, 65535).astype(np.uint16)
        u[rng.random((self.H, self.W)) < hole_frac] = 0
        return u

    def cloud(self, t: int) -> np.ndarray:
        """float32 4 x N planar: a Velodyne-like fan of rays hitting the plane z = Z (camera frame)."""
        rng = np.random.default_rng(self.seed * 7919 + t)
        # sample directions over the camera's field of view (plus margin), ring-major
        v = np.linspace(-0.50, 0.40, self.n_rings)[:, None]          # tan(elevation) in camera y (image covers +-0.26)
        u = np.linspace(-3.0, 3.0, self.n_az)[None, :]               # tan(azimuth) in camera x (image covers +-0.85): ~16 % land inside
        X = (u * self.Z) * np.ones_like(v); Y = (v * self.Z) * np.ones_like(u); Zc = np.full_like(X, self.Z)
        Zc = Zc + rng.normal(0.0, 0.01, Zc.shape)
        cam = np.stack([X.ravel(), Y.ravel(), Zc.ravel(), np.ones(X.size)])
        velo = self.Tr_inv @ cam
        pts = np.stack([velo[0], velo[1], velo[2], np.ones(X.size)]).astype(np.float32)
        return np.ascontiguousarray(pts)


def distort_normalized(x, y, dist):
    """OpenCV's distortion model (k1, k2, p1, p2[, k3]) on normalised camera coordinates -> distorted normalised coordinates"""
    k1, k2, p1, p2 = dist[:4]
    k3 = dist[4] if len(dist) > 4 else 0.0
    r2 = x * x + y * y
    radial = 1 + r2 * (k1 + r2 * (k2 + r2 * k3))
    return x * radial + 2 * p1 * x * y + p2 * (r2 + 2 * x * x), y * radial + p1 * (r2 + 2 * y * y) + 2 * p2 * x * y


def rectification_maps(W: int, H: int, cam, dist, R=None):
    """float32 (map_x, map_y), H x W, of cv::initUndistortRectifyMap(K, dist, R, K, (W, H), CV_32FC1), K = (fx, fy, cx, cy): for each
    rectified pixel (u, v) the raw (distorted) pixel it samples.  R = None: the identity."""
    fx, fy, cx, cy = (float(v) for v in cam)
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    ray = np.stack([(u - cx) / fx, (v - cy) / fy, np.ones_like(u)])
    if R is not None:
        ray = np.tensordot(np.asarray(R, np.float64).T, ray, 1)         # R^-1 = R^T
    xd, yd = distort_normalized(ray[0] / ray[2], ray[1] / ray[2], np.asarray(dist, np.float64))
    return (xd * fx + cx).astype(np.float32), (yd * fy + cy).astype(np.float32)


def undistorted_pixel_map(W: int, H: int, cam, dist, iterations: int = 100):
    """For every pixel (u, v) of a W x H distorted image: the pixel of the undistorted (pinhole) image it shows, (map_x, map_y) float64 H x W.
    The inverse of the distortion model by fixed-point iteration, run until it has converged (checked by distorting the result again)."""
    fx, fy, cx, cy = (float(v) for v in cam)
    dist = np.asarray(dist, np.float64)
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    xd, yd = (u - cx) / fx, (v - cy) / fy
    x, y = xd.copy(), yd.copy()
    for _ in range(iterations):
        dx, dy = distort_normalized(x, y, dist)
        x, y = x + (xd - dx), y + (yd - dy)
    dx, dy = distort_normalized(x, y, dist)
    err = max(np.abs(dx - xd).max() * fx, np.abs(dy - yd).max() * fy)
    if not err < 1e-6:
        raise ValueError(f"the inverse distortion did not converge ({err} px)")
    return x * fx + cx, y * fy + cy


def stereo_disparity_field(W: int = KITTI_W, H: int = KITTI_H) -> np.ndarray:
    """Smooth, NON-uniform disparity (pixels) of a rectified pair, defined on the right image: near ground at the bottom of the image
    (large disparity), far scene at the top, plus a slow lateral modulation.  4 ... ~30 px at KITTI size (= 97 m ... 13 m at bf 387)."""
    y = np.linspace(0.0, 1.0, H)[:, None]
    x = np.arange(W)[None, :]
    return 4.0 + 22.0 * y * y + 3.0 * np.sin(x / 90.0) * (0.3 + y)


def stereo_pair(seed: int, W: int = KITTI_W, H: int = KITTI_H):
    """(left, right) uint8 images of a rectified stereo rig (BASELINE config C, SURVEY 8(d)): right(x, y) = left(x + d(x, y), y),
    bilinearly resampled, d = stereo_disparity_field; so a left keypoint at uL has its match near uL - d."""
    margin = 48
    tex = make_image(seed, W + margin, H).astype(np.float64)
    left = tex[:, :W]
    d = stereo_disparity_field(W, H)
    xs = np.arange(W)[None, :] + d
    x0 = np.floor(xs).astype(np.int64); fx = xs - x0
    x0 = np.clip(x0, 0, W + margin - 2)
    rows = np.arange(H)[:, None]
    right = tex[rows, x0] * (1.0 - fx) + tex[rows, x0 + 1] * fx
    return np.ascontiguousarray(np.clip(np.rint(left), 0, 255).astype(np.uint8)), np.ascontiguousarray(np.clip(np.rint(right), 0, 255).astype(np.uint8))


# ---- synthetic local-BA problems (flat graph as the C-ABI shim gathers it from Optimizer::LocalBundleAdjustment, src/Optimizer.cc:1116-1404):
# key-frame poses along a forward trajectory with yaw, points in front of them, mono / stereo observations with pixel noise per octave,
# a few gross outliers, perturbed initial estimates; the first key frames are fixed.
def _quat_yaw(a):
    return np.array([0.0, np.sin(a / 2), 0.0, np.cos(a / 2)])       # rotation about the camera y axis (x, y, z, w)


def _rot(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def make_ba_problem(seed, n_kf=8, n_fixed=2, n_points=600, outlier_frac=0.03, stereo_frac=0.6, pose_noise=(0.004, 0.03), point_noise=0.06):
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy, bf = KITTI_FX, KITTI_FY, KITTI_CX, KITTI_CY, KITTI_BF
    W, H = KITTI_W, KITTI_H
    # true poses Tcw: camera moves forward (world z) with a slow yaw
    true_poses = []
    for k in range(n_kf):
        q = _quat_yaw(0.01 * k)
        cpos = np.array([0.05 * k, 0.0, 0.9 * k])                    # camera centre in the world
        R = _rot(q)
        t = -R @ cpos
        true_poses.append(np.concatenate([q, t]))
    true_poses = np.array(true_poses)
    pts = np.column_stack([rng.uniform(-12, 12, n_points), rng.uniform(-2.5, 1.5, n_points), rng.uniform(6, 45, n_points) + 0.9 * n_kf * rng.random(n_points)])
    e_point, e_pose, obs, stereo, inv_s2, is_out = [], [], [], [], [], []
    for j in range(n_points):
        for k in range(n_kf):
            R = _rot(true_poses[k, :4]); pc = R @ pts[j] + true_poses[k, 4:]
            if pc[2] < 1.0:
                continue
            u = fx * pc[0] / pc[2] + cx; v = fy * pc[1] / pc[2] + cy
            if not (20 < u < W - 20 and 20 < v < H - 20) or rng.random() < 0.15:
                continue
            octave = int(rng.integers(0, 8)); sig = 1.2 ** octave
            st = rng.random() < stereo_frac
            out = rng.random() < outlier_frac
            nu, nv = rng.normal(0, 0.6 * sig, 2)
            if out:
                nu += rng.choice([-1, 1]) * rng.uniform(15, 60); nv += rng.choice([-1, 1]) * rng.uniform(10, 40)
            ur = (u - bf / pc[2] + rng.normal(0, 0.6 * sig)) if st else -1.0
            if ur < 0:                 # the reference tells a stereo observation by mvuRight >= 0 (src/Optimizer.cc:1286-1311)
                st, ur = False, -1.0
            e_point.append(j); e_pose.append(k); obs.append([u + nu, v + nv, ur]); stereo.append(st); inv_s2.append(1.0 / (sig * sig)); is_out.append(out)
    # Optimizer::LocalBundleAdjustment only adjusts points seen from a LOCAL (non-fixed) key frame (src/Optimizer.cc:1133-1160): drop the
    # others, as the gathering shim would
    e_point = np.array(e_point, np.int64); e_pose = np.array(e_pose, np.int64)
    local = np.zeros(n_points, bool); local[e_point[e_pose >= n_fixed]] = True
    if n_fixed >= n_kf:
        local[:] = True          # no local key frame at all (structure-only adjustment): keep the graph as generated
    keep_e = local[e_point]
    remap = np.cumsum(local) - 1
    e_point = remap[e_point[keep_e]]; e_pose = e_pose[keep_e]
    obs = [o for o, k in zip(obs, keep_e) if k]; stereo = [o for o, k in zip(stereo, keep_e) if k]
    inv_s2 = [o for o, k in zip(inv_s2, keep_e) if k]; is_out = [o for o, k in zip(is_out, keep_e) if k]
    pts = pts[local]
    init_poses = true_poses.copy()
    for k in range(n_fixed, n_kf):
        dq = np.concatenate([rng.normal(0, pose_noise[0], 3), [1.0]]); dq /= np.linalg.norm(dq)
        x1, y1, z1, w1 = dq; x2, y2, z2, w2 = init_poses[k, :4]
        q = np.array([w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2, w1 * y2 + y1 * w2 + z1 * x2 - x1 * z2, w1 * z2 + z1 * w2 + x1 * y2 - y1 * x2, w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2])
        init_poses[k, :4] = q / np.linalg.norm(q)
        init_poses[k, 4:] += rng.normal(0, pose_noise[1], 3)
    init_pts = pts + rng.normal(0, point_noise, pts.shape)
    fixed = np.zeros(n_kf, np.uint8); fixed[:n_fixed] = 1
    return dict(poses=init_poses.astype(np.float32), pose_fixed=fixed, points=init_pts.astype(np.float32),
                e_point=np.array(e_point, np.int32), e_pose=np.array(e_pose, np.int32), obs=np.array(obs, np.float32),
                stereo=np.array(stereo, np.uint8), inv_sigma2=np.array(inv_s2, np.float32), cam=(fx, fy, cx, cy, bf),
                true_poses=true_poses, true_points=pts, is_outlier=np.array(is_out, bool))


def ba_args(p):
    return (p["poses"], p["pose_fixed"], p["points"], p["e_point"], p["e_pose"], p["obs"], p["stereo"], p["inv_sigma2"], *p["cam"])


# ---- PNG streams (the input of cv::imread at Examples/RGB-L/rgbl_kitti.cc:87) -------------------------------------------------------
def encode_png(img: np.ndarray, filters=None, idat_chunk: int = 1 << 16, level: int = 6) -> bytes:
    """A PNG file (8-bit gray / RGB / RGBA, non-interlaced) of `img` (H x W or H x W x {3,4}, samples in FILE order R, G, B[, A]).
    `filters`: one filter type 0..4 (None, Sub, Up, Average, Paeth) per row, default = all five cycling, so that decoders are
    exercised on every type; the zlib stream is split over IDAT chunks of `idat_chunk` bytes."""
    import struct
    import zlib
    img = np.ascontiguousarray(img, np.uint8)
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else img.shape[2]
    ctype = {1: 0, 3: 2, 4: 6}[ch]
    rows = img.reshape(h, w * ch).astype(np.int16)
    if filters is None:
        filters = np.arange(h) % 5
    filters = np.asarray(filters, np.int64)
    a = np.zeros_like(rows); a[:, ch:] = rows[:, :-ch]                       # left
    b = np.zeros_like(rows); b[1:] = rows[:-1]                               # up
    c = np.zeros_like(rows); c[1:, ch:] = rows[:-1, :-ch]                    # upper left
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    paeth = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
    pred = np.stack([np.zeros_like(rows), a, b, (a + b) >> 1, paeth])[filters, np.arange(h)]
    raw = np.empty((h, w * ch + 1), np.uint8)
    raw[:, 0] = filters
    raw[:, 1:] = ((rows - pred) & 0xff).astype(np.uint8)
    z = zlib.compress(raw.tobytes(), level)

    def chunk(tag: bytes, data: bytes) -> bytes:
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xffffffff)

    out = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, ctype, 0, 0, 0))
    for i in range(0, len(z), idat_chunk):
        out += chunk(b"IDAT", z[i:i + idat_chunk])
    return out + chunk(b"IEND", b"")


def colorize(gray: np.ndarray, seed: int = 0, alpha: bool = False) -> np.ndarray:
    """A colour image (file order R, G, B[, A]) whose channels are different smooth remappings of a synthetic gray image."""
    rng = np.random.default_rng(seed)
    g = gray.astype(np.float64)
    H, W = gray.shape
    tint = [_upsample_bilinear(rng.random((max(2, H // 64 + 2), max(2, W // 64 + 2))), H, W) for _ in range(3)]
    chans = [np.clip(g * (0.6 + 0.8 * t) + 20.0 * (t - 0.5), 0, 255).astype(np.uint8) for t in tint]
    if alpha:
        chans.append(rng.integers(0, 256, gray.shape, dtype=np.uint8))
    return np.stack(chans, -1)


def encode_png16(img: np.ndarray, filters=None, idat_chunk: int = 1 << 16, level: int = 6) -> bytes:
    """A 16-bit PNG file (gray, or RGB for an H x W x 3 array; non-interlaced) of the uint16 `img`, samples stored big-endian: what an
    RGB-D sensor's depth PNG holds.  `filters` and `idat_chunk` as for encode_png; the filters work byte-wise with 2 bytes per sample."""
    import struct
    import zlib
    img = np.ascontiguousarray(img, np.uint16)
    h, w = img.shape[:2]
    ch = 1 if img.ndim == 2 else img.shape[2]
    bpp = 2 * ch
    rows = img.astype(">u2").view(np.uint8).reshape(h, w * bpp).astype(np.int16)
    if filters is None:
        filters = np.arange(h) % 5
    filters = np.asarray(filters, np.int64)
    a = np.zeros_like(rows); a[:, bpp:] = rows[:, :-bpp]
    b = np.zeros_like(rows); b[1:] = rows[:-1]
    c = np.zeros_like(rows); c[1:, bpp:] = rows[:-1, :-bpp]
    p = a + b - c
    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
    paeth = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
    pred = np.stack([np.zeros_like(rows), a, b, (a + b) >> 1, paeth])[filters, np.arange(h)]
    raw = np.empty((h, w * bpp + 1), np.uint8)
    raw[:, 0] = filters
    raw[:, 1:] = ((rows - pred) & 0xff).astype(np.uint8)
    z = zlib.compress(raw.tobytes(), level)

    def chunk(tag: bytes, data: bytes) -> bytes:
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xffffffff)

    out = b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 16, {1: 0, 3: 2}[ch], 0, 0, 0))
    for i in range(0, len(z), idat_chunk):
        out += chunk(b"IDAT", z[i:i + idat_chunk])
    return out + chunk(b"IEND", b"")

"""Colour camera input on the GPU (rgbl_set_input_channels: the cvtColor of Tracking::GrabImageRGBL / GrabImageRGBD / GrabImageStereo) at
sizes users run: KITTI-like 1241x376 RGB-L frames, TUM-like 640x480 RGB-D frames with a distorted camera, 1280x720 stereo pairs tracked
at 640x360 (input resize) and the raw pairs of the EuRoC-like rig (rectification), from arrays and colour PNGs.  The frames (level 0,
keypoints, descriptors, mvDepth, mvuRight) equal bit for bit those of a gray context fed the images cv2 converts (after cv2's resize or
remap of the colour image, as the reference does); the three sequence runners, host and resident mode, give bitwise the poses, matches
and inliers of the same runner fed host-converted images.  Rehearsable on the CPU against the emulated library (RGBL_LIB_PATH,
tests/cuda_emu/build.py)."""
import numpy as np
import pytest

from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S

pytestmark = pytest.mark.gpu

cv2 = pytest.importorskip("cv2")

SW, SH = 1280, 720
FULL_CAM = (700.0, 700.0, 640.0, 360.0, 360.0)


def colour(gray, seed, alpha=False):
    return np.ascontiguousarray(S.colorize(gray, seed, alpha))


def to_gray(img, rgb=True, size=None, maps=None):
    """the reference's Grab*: resize (size) or remap (maps) of the colour image, then cvtColor with channel 0 red (rgb) or blue"""
    if maps is not None:
        img = cv2.remap(img, maps[0], maps[1], cv2.INTER_LINEAR)
    elif size is not None:
        img = cv2.resize(img, size, interpolation=cv2.INTER_LINEAR)
    ch = img.shape[2]
    code = {(3, True): cv2.COLOR_RGB2GRAY, (3, False): cv2.COLOR_BGR2GRAY, (4, True): cv2.COLOR_RGBA2GRAY, (4, False): cv2.COLOR_BGRA2GRAY}
    return cv2.cvtColor(img, code[(ch, rgb)])


def _level0(c, n):
    out = []
    for f in range(n):
        img = np.empty((c.height, c.width), np.uint8)
        F.check(L.lib().rgbl_orb_get_level(c.handle, f, 0, L.ptr(img), c.width, None, None), c.handle)
        out.append(img.tobytes())
    return out


def _frames(b, c):
    fr = b.download()
    assert min(len(f[0]) for f in fr) > 100
    return [np.array(a).tobytes() for f in fr for a in f] + _level0(c, b.nF)


def _ctx(w, h, T, channels=1, camera_rgb=True, resize_to=None, maps=None, max_points=0):
    c = F.Context(w, h, 2000, max_batch=2 * T, max_points=max_points)
    if resize_to:
        c.set_input_resize(*resize_to)
    if maps is not None:
        c.set_stereo_rectification(*maps, *maps)
    c.set_input_channels(channels, camera_rgb)
    return c


def test_rgbl_kitti_colour_frames():
    T = 4
    s = S.PlaneSequence(11, T)
    imgs = [colour(s.image(t), t) for t in range(T)]
    clouds = [s.cloud(t) for t in range(T)]
    prm = F.make_depth_params(bf=s.cam[4])
    c0 = _ctx(s.W, s.H, T, max_points=clouds[0].shape[1])
    try:
        b0 = F.RgblBatch(c0, [to_gray(i) for i in imgs], clouds, s.P, prm, pinned=False)
        b0.upload(); b0.process_resident()
        want = _frames(b0, c0)
        b0.set_inputs([to_gray(i, False) for i in imgs], clouds)          # a PNG file holds R, G, B: Camera.RGB = 1 weights R as blue
        b0.upload(); b0.process_resident()
        want_png = _frames(b0, c0)
    finally:
        c0.close()
    c = _ctx(s.W, s.H, T, 3, True, max_points=clouds[0].shape[1])
    try:
        b = F.RgblBatch(c, imgs, clouds, s.P, prm, pinned=False)
        b.upload(); b.process_resident()
        assert _frames(b, c) == want
        b.upload_kitti_png([S.encode_png(i) for i in imgs], [np.ascontiguousarray(p.T) for p in clouds], camera_rgb=True)
        b.process_resident()
        assert _frames(b, c)[-T:] == want_png[-T:]           # level 0 (the clouds went in as KITTI records)
    finally:
        c.close()


def test_rgbd_tum_colour_frames_with_a_distorted_camera():
    T, W, H = 4, S.TUM_W, S.TUM_H
    cam = (S.TUM1_FX, S.TUM1_FY, S.TUM1_CX, S.TUM1_CY, S.TUM1_BF)
    s = S.PlaneSequence(23, T, W=W, H=H, cam=cam, Z=3.0)
    imgs = [colour(s.image(t), t, alpha=True) for t in range(T)]             # RGBA, BGR order (Camera.RGB = 0)
    deps = [s.depth16(t, S.TUM_DEPTH_FACTOR) for t in range(T)]
    scale = F.depth_map_factor(S.TUM_DEPTH_FACTOR)
    out = []
    for ch in (1, 4):
        c = _ctx(W, H, T, ch, False)
        try:
            c.set_camera_distortion(*cam[:4], S.TUM1_DIST)
            b = F.RgbdBatch(c, imgs if ch == 4 else [to_gray(i, False) for i in imgs], deps, pinned=False)
            b.upload(); b.process_resident(scale, cam[4])
            out.append(_frames(b, c) + [k.tobytes() for k in b.download_keys_un()])
        finally:
            c.close()
    assert out[0] == out[1]


def scaled_cam(w, h):
    sx, sy = np.float32(w / SW), np.float32(h / SH)
    fx, fy, cx, cy, bf = (np.float32(v) for v in FULL_CAM)
    return float(fx * sx), float(fy * sy), float(cx * sx), float(cy * sy), float(bf * sx)


def _stereo_frames(c, lefts, rights, cam, png=False):
    mb, mbf = float(np.float32(cam[4]) / np.float32(cam[0])), cam[4]
    b = F.StereoBatch(c, lefts, rights, pinned=False)
    if png:
        b.upload_png([S.encode_png(i) for i in lefts], [S.encode_png(i) for i in rights], camera_rgb=True)
    else:
        b.upload()
    b.process_resident(mb, mbf)
    return _frames(b, c)


def test_stereo_colour_pairs_with_the_resize():
    T, w, h = 3, 640, 360
    s = S.PlaneSequence(61, T, shift_px=14, W=SW, H=SH, cam=FULL_CAM)
    lefts, rights = [colour(s.image(t), t) for t in range(T)], [colour(s.right_image(t), t + 9) for t in range(T)]
    cam = scaled_cam(w, h)
    c0 = _ctx(w, h, T)
    try:
        want = _stereo_frames(c0, [to_gray(i, True, (w, h)) for i in lefts], [to_gray(i, True, (w, h)) for i in rights], cam)
        want_png = _stereo_frames(c0, [to_gray(i, False, (w, h)) for i in lefts], [to_gray(i, False, (w, h)) for i in rights], cam)
    finally:
        c0.close()
    c = _ctx(w, h, T, 3, True, (SW, SH))
    try:
        assert _stereo_frames(c, lefts, rights, cam) == want
        assert _stereo_frames(c, lefts, rights, cam, png=True) == want_png
    finally:
        c.close()


def test_stereo_euroc_colour_pairs_with_rectification():
    T = 3
    s = S.PlaneSequence(5, T, W=S.EUROC_W, H=S.EUROC_H, cam=S.EUROC_CAM, dist=S.EUROC_DIST)
    maps = s.rectification_maps()
    lefts, rights = [colour(s.raw_left_image(t), t) for t in range(T)], [colour(s.raw_right_image(t), t + 9) for t in range(T)]
    c0 = _ctx(s.W, s.H, T)
    try:
        want = _stereo_frames(c0, [to_gray(i, True, maps=maps) for i in lefts], [to_gray(i, True, maps=maps) for i in rights], s.cam)
        want_png = _stereo_frames(c0, [to_gray(i, False, maps=maps) for i in lefts], [to_gray(i, False, maps=maps) for i in rights], s.cam)
    finally:
        c0.close()
    c = _ctx(s.W, s.H, T, 3, True, maps=maps)
    try:
        assert _stereo_frames(c, lefts, rights, s.cam) == want
        assert _stereo_frames(c, lefts, rights, s.cam, png=True) == want_png
    finally:
        c.close()


def _runner(kind, s, T, nB, colour_in, resident):
    """the sequence of `kind` through its runner: colour images converted on the device (colour_in), or host-converted gray images"""
    conv = (lambda a: a) if colour_in else to_gray
    c = _ctx(s.W, s.H, T, 3 if colour_in else 1, True, max_points=s.cloud(0).shape[1] if kind == "rgbl" else 0)
    ch = 3 if colour_in else 1
    try:
        if kind == "rgbl":
            r = F.SequenceRunner(c, s.P, F.make_depth_params(bf=s.cam[4]), T, s.W, s.H, s.cloud(0).shape[1], nB, pinned=False, channels=ch)
        elif kind == "rgbd":
            r = F.SequenceRunner.rgbd(c, F.depth_map_factor(256.0), s.cam[4], T, s.W, s.H, nB, pinned=False, channels=ch)
        else:
            r = F.SequenceRunner.stereo(c, float(np.float32(s.cam[4]) / np.float32(s.cam[0])), s.cam[4], T, s.W, s.H, nB, pinned=False, channels=ch)
        for m in range(nB):
            ts = range(m * T, (m + 1) * T)
            second = ([s.cloud(t) for t in ts] if kind == "rgbl" else [s.depth16(t, 256.0) for t in ts] if kind == "rgbd"
                      else [conv(colour(s.right_image(t), t + 9)) for t in ts])
            r.set_batch(m, [conv(colour(s.image(t), t)) for t in ts], second)
            if resident:
                r.stage(m, m)
        th_last, th_local = (7.0, 1.0) if kind == "stereo" else (15.0, 3.0)
        cp = F.make_chain_params(s.pose(0), *s.cam, th_last=th_last, local_map_frames=2, th_local=th_local)
        o = r.run(cp, nB, first=0, resident_slots=nB if resident else 0, want_frames=True)
        return {k: np.array(v) for k, v in o.items()}
    finally:
        c.close()


@pytest.mark.parametrize("kind", ["rgbl", "rgbd", "stereo"])
def test_sequence_runners_with_colour_input_equal_host_converted_runners(kind):
    T, nB = 4, 3
    s = S.PlaneSequence(31, T * nB, shift_px=7, W=640, H=376)
    want = _runner(kind, s, T, nB, False, False)
    assert (want["n_inliers"][1:] > 50).all()
    for resident in (False, True):
        got = _runner(kind, s, T, nB, True, resident)
        for k in want:
            assert got[k].tobytes() == want[k].tobytes(), (kind, resident, k)

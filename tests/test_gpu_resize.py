"""The input resize on the device (rgbl_set_input_resize: System::TrackRGBD's / TrackStereo's cv::resize to Settings' new image size):
RGB-D and stereo frames built from input-size images equal, bitwise, the frames of a context without the resize fed cv2-resized inputs,
and the oracle's frames; resize and rectification together equal one remap of the input-size images; the RGB-D and stereo sequence
runners (host, resident and PNG inputs) give the poses, matches and inliers of the same runner on host-resized inputs; and a setting that
was cleared again leaves every input kind as a fresh context has it."""
import ctypes as C

import numpy as np
import pytest

import oracle
from oracle import rectify as RC
from oracle import rgbd as ORGBD
from oracle import stereo as OST
import tracking_data as TD
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S

pytestmark = pytest.mark.gpu

SW, SH = 1280, 720                        # the camera's size (a RealSense-like stream)
FULL_CAM = (700.0, 700.0, 640.0, 360.0, 360.0)            # fx, fy, cx, cy, bf at the camera's size (18 px disparity)
FACTOR = 256.0                            # RGBD.DepthMapFactor of the depth images


def scaled_cam(w, h):
    """Settings' intrinsics at the new size: fx, cx by w / SW, fy, cy by h / SH, bf = b * fx"""
    sx, sy = np.float32(w / SW), np.float32(h / SH)
    fx, fy, cx, cy, bf = (np.float32(v) for v in FULL_CAM)
    return float(fx * sx), float(fy * sy), float(cx * sx), float(cy * sy), float(bf * sx)


def seq(n):
    return S.PlaneSequence(61, n, shift_px=14, W=SW, H=SH, cam=FULL_CAM)


def resize(img, w, h):
    import cv2
    return cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR)


def _level0(c, n):
    out = []
    for f in range(n):
        img = np.empty((c.height, c.width), np.uint8)
        F.check(L.lib().rgbl_orb_get_level(c.handle, f, 0, L.ptr(img), c.width, None, None), c.handle)
        out.append(img)
    return out


def _frames(b, c):
    return [np.array(a).tobytes() for fr in b.download() for a in fr] + [l.tobytes() for l in _level0(c, b.nF)]


def _ctx(w, h, T, resize_to=None):
    c = F.Context(w, h, 2000, max_batch=2 * T)
    if resize_to:
        c.set_input_resize(*resize_to)
    return c


def _same_as_oracle(got, ref):
    k, d, dep, ur = (np.array(a) for a in got)
    assert len(k) == len(ref["k"])
    for name in k.dtype.names:
        assert k[name].tobytes() == ref["k"][name].tobytes(), name
    assert d.tobytes() == ref["d"].tobytes() and dep.tobytes() == ref["depth"].tobytes() and ur.tobytes() == ref["ur"].tobytes()


def test_rgbd_frames_equal_host_resized_frames_and_the_oracle():
    pytest.importorskip("cv2")
    T, w, h = 4, 640, 360
    s = seq(T)
    imgs, deps = [s.image(t) for t in range(T)], [s.depth16(t, FACTOR) for t in range(T)]
    scale, bf = F.depth_map_factor(FACTOR), scaled_cam(w, h)[4]
    c0 = _ctx(w, h, T)
    try:
        b0 = F.RgbdBatch(c0, [resize(i, w, h) for i in imgs], [resize(d, w, h) for d in deps], pinned=False)
        b0.upload(); b0.process_resident(scale, bf)
        want = _frames(b0, c0)
        host = [tuple(np.array(a) for a in fr) for fr in b0.download()]
    finally:
        c0.close()
    c = _ctx(w, h, T, (SW, SH))
    try:
        b = F.RgbdBatch(c, imgs, deps, pinned=False)
        b.upload(); b.process_resident(scale, bf)
        assert _frames(b, c) == want
        b.upload_png([S.encode_png(i) for i in imgs], [S.encode_png16(d) for d in deps])
        b.process_resident(scale, bf)
        assert _frames(b, c) == want
    finally:
        c.close()
    ex = oracle.Extractor(2000)
    for t in range(T):
        ref = ORGBD.rgbd_frame(ex, resize(imgs[t], w, h), resize(deps[t], w, h), ORGBD.depth_map_factor(FACTOR), bf)
        _same_as_oracle(host[t], ref)
        assert (ref["depth"] > 0).sum() > 100


@pytest.mark.parametrize("w,h", [(960, 540), (640, 360)], ids=["factor1.33", "factor2"])
def test_stereo_frames_equal_host_resized_frames_and_the_oracle(w, h):
    pytest.importorskip("cv2")
    T = 3
    s = seq(T)
    lefts, rights = [s.image(t) for t in range(T)], [s.right_image(t) for t in range(T)]
    _, _, _, _, mbf = scaled_cam(w, h)
    mb = float(np.float32(mbf) / np.float32(scaled_cam(w, h)[0]))
    c0 = _ctx(w, h, T)
    try:
        b0 = F.StereoBatch(c0, [resize(i, w, h) for i in lefts], [resize(i, w, h) for i in rights], pinned=False)
        b0.upload(); b0.process_resident(mb, mbf)
        want = _frames(b0, c0)
        host = [tuple(np.array(a) for a in fr) for fr in b0.download()]
    finally:
        c0.close()
    c = _ctx(w, h, T, (SW, SH))
    try:
        b = F.StereoBatch(c, lefts, rights, pinned=False)
        b.upload(); b.process_resident(mb, mbf)
        assert _frames(b, c) == want
        b.upload_png([S.encode_png(i) for i in lefts], [S.encode_png(i) for i in rights])
        b.process_resident(mb, mbf)
        assert _frames(b, c) == want
    finally:
        c.close()
    exl, exr = oracle.Extractor(2000), oracle.Extractor(2000)
    for t in range(T):
        ref = OST.stereo_frame(exl, exr, resize(lefts[t], w, h), resize(rights[t], w, h), mb, mbf)
        _same_as_oracle(host[t], ref)
        assert (ref["depth"] > 0).sum() > 100


def test_resize_with_rectification_is_one_remap():
    """maps at the context's size whose coordinates index the camera-size images (initUndistortRectifyMap(..., newImSize)): the stereo
    frames equal those of a context without either setting fed cv2.remap of the camera-size images"""
    T, w, h = 2, 960, 540
    s = seq(T)
    lefts, rights = [s.image(t) for t in range(T)], [s.right_image(t) for t in range(T)]
    xs, ys = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    r2 = ((xs - w / 2) ** 2 + (ys - h / 2) ** 2) / (w * w)
    mx = np.ascontiguousarray(((xs + 0.5) * SW / w - 0.5) * (1 - 0.02 * r2) + 6.0, np.float32)
    my = np.ascontiguousarray(((ys + 0.5) * SH / h - 0.5) * (1 - 0.02 * r2) + 3.0, np.float32)
    _, _, _, _, mbf = scaled_cam(w, h)
    mb = float(np.float32(mbf) / np.float32(scaled_cam(w, h)[0]))
    c0 = _ctx(w, h, T)
    try:
        b0 = F.StereoBatch(c0, [RC.remap(i, mx, my) for i in lefts], [RC.remap(i, mx, my) for i in rights], pinned=False)
        b0.upload(); b0.process_resident(mb, mbf)
        want = _frames(b0, c0)
    finally:
        c0.close()
    c = _ctx(w, h, T, (SW, SH))
    try:
        c.set_stereo_rectification(mx, my, mx, my)
        b = F.StereoBatch(c, lefts, rights, pinned=False)
        b.upload(); b.process_resident(mb, mbf)
        assert _frames(b, c) == want
        b.upload_png([S.encode_png(i) for i in lefts], [S.encode_png(i) for i in rights])
        b.process_resident(mb, mbf)
        assert _frames(b, c) == want
    finally:
        c.close()


def _runner(kind, s, T, nB, w, h, resize_on, resident):
    c = _ctx(w, h, T, (SW, SH) if resize_on else None)
    cam = scaled_cam(w, h)
    try:
        iw, ih = (SW, SH) if resize_on else (w, h)
        conv = (lambda a: a) if resize_on else (lambda a: resize(a, w, h))
        if kind == "rgbd":
            r = F.SequenceRunner.rgbd(c, F.depth_map_factor(FACTOR), cam[4], T, iw, ih, nB, pinned=False)
        else:
            r = F.SequenceRunner.stereo(c, float(np.float32(cam[4]) / np.float32(cam[0])), cam[4], T, iw, ih, nB, pinned=False)
        for m in range(nB):
            ts = range(m * T, (m + 1) * T)
            second = [s.depth16(t, FACTOR) for t in ts] if kind == "rgbd" else [s.right_image(t) for t in ts]
            r.set_batch(m, [conv(s.image(t)) for t in ts], [conv(a) for a in second])
            if resident:
                r.stage(m, m)
        cp = F.make_chain_params(s.pose(0), *cam, th_last=7.0, local_map_frames=2, th_local=1.0)
        o = r.run(cp, nB, first=0, resident_slots=nB if resident else 0, want_frames=True)
        return {k: np.array(v) for k, v in o.items()}
    finally:
        c.close()


def _png_chain(kind, s, T, nB, w, h, resize_on):
    """the same sequence through the batch API, images (and depth images) as PNG files"""
    c = _ctx(w, h, T, (SW, SH) if resize_on else None)
    cam = scaled_cam(w, h)
    conv = (lambda a: a) if resize_on else (lambda a: resize(a, w, h))
    out = []
    try:
        for m in range(nB):
            ts = list(range(m * T, (m + 1) * T))
            imgs = [conv(s.image(t)) for t in ts]
            if kind == "rgbd":
                deps = [conv(s.depth16(t, FACTOR)) for t in ts]
                b = F.RgbdBatch(c, imgs, deps, pinned=False)
                b.upload_png([S.encode_png(i) for i in imgs], [S.encode_png16(d) for d in deps])
                b.process_resident(F.depth_map_factor(FACTOR), cam[4])
            else:
                rights = [conv(s.right_image(t)) for t in ts]
                b = F.StereoBatch(c, imgs, rights, pinned=False)
                b.upload_png([S.encode_png(i) for i in imgs], [S.encode_png(i) for i in rights])
                b.process_resident(float(np.float32(cam[4]) / np.float32(cam[0])), cam[4])
            b.track_begin2(F.make_chain_params(s.pose(0), *cam, th_last=7.0, continue_sequence=m > 0, local_map_frames=2, th_local=1.0))
            out.append({k: np.array(v) for k, v in b.track_end2().items()})
    finally:
        c.close()
    return out


@pytest.mark.parametrize("kind", ["rgbd", "stereo"])
def test_sequence_runner_with_resize_equals_host_resized_runner(kind):
    pytest.importorskip("cv2")
    T, nB, w, h = 4, 3, 640, 360
    s = seq(T * nB)
    want = _runner(kind, s, T, nB, w, h, False, False)
    assert (want["n_inliers"][1:] > 50).all()
    for resident in (False, True):
        got = _runner(kind, s, T, nB, w, h, True, resident)
        for k in want:
            assert got[k].tobytes() == want[k].tobytes(), (kind, resident, k)
    want_png = _png_chain(kind, s, T, nB, w, h, False)
    got_png = _png_chain(kind, s, T, nB, w, h, True)
    for a, b in zip(want_png, got_png):
        for k in a:
            assert a[k].tobytes() == b[k].tobytes(), (kind, "png", k)


def _all_kinds(c, s, T):
    """a stereo batch, an RGB-L chain and an RGB-D batch at the context's own size -> every output"""
    out = []
    sb = F.StereoBatch(c, [s.image(t) for t in range(T)], [s.right_image(t) for t in range(T)], pinned=False)
    sb.upload(); sb.process_resident(float(np.float32(S.KITTI_BF) / np.float32(S.KITTI_FX)), S.KITTI_BF)
    out.append([np.array(a) for fr in sb.download() for a in fr])
    rb = F.RgblBatch(c, [s.image(t) for t in range(T)], [s.cloud(t) for t in range(T)], s.P, F.make_depth_params(bf=S.KITTI_BF), pinned=False)
    rb.upload(); rb.process_resident()
    out.append([np.array(a) for fr in rb.download() for a in fr])
    rb.track_begin2(F.make_chain_params(s.pose(0), *TD.CAM, local_map_frames=2))
    out.append(list(rb.track_end2().values()))
    db = F.RgbdBatch(c, [s.image(t) for t in range(T)], [s.depth16(t) for t in range(T)], pinned=False)
    db.upload(); db.process_resident(F.depth_map_factor(256), S.KITTI_BF)
    out.append([np.array(a) for fr in db.download() for a in fr])
    return out


def test_resize_off_is_unchanged():
    """the resize set, used and cleared: stereo, RGB-L and RGB-D results are bitwise those of a context that never had it"""
    T = 3
    s = S.PlaneSequence(43, T + 1)
    mk = lambda: F.Context(S.KITTI_W, S.KITTI_H, 2000, max_batch=2 * T, max_points=s.cloud(0).shape[1])
    c = mk()
    try:
        ref = _all_kinds(c, s, T)
    finally:
        c.close()
    c = mk()
    try:
        c.set_input_resize(2 * S.KITTI_W, 2 * S.KITTI_H)
        big = [np.ascontiguousarray(np.repeat(np.repeat(s.image(t), 2, 0), 2, 1)) for t in range(T)]
        sb = F.StereoBatch(c, big, big, pinned=False)
        sb.upload(); sb.process_resident(0.5, 40.0)
        c.set_input_resize(0, 0)
        got = _all_kinds(c, s, T)
    finally:
        c.close()
    for a, b in zip(ref, got):
        for p, q in zip(a, b):
            assert p.tobytes() == q.tobytes()


def test_resize_refusals_on_the_device():
    """the rules of rgbl_set_input_resize on a real context (the full set runs under emulation in test_input_resize_emu.py)"""
    c = _ctx(640, 360, 2)
    lib, h = L.lib(), c.handle
    try:
        assert lib.rgbl_set_input_resize(h, 639, 720) == L.RGBL_E_UNSUPPORTED
        assert lib.rgbl_set_input_resize(h, 1280, 0) == L.RGBL_E_INVALID
        c.set_input_resize(1000, 600)                                   # not integer factors: stereo only
        s = seq(2)
        imgs = [resize(s.image(t), 1000, 600) for t in range(2)]
        with pytest.raises(L.RgblError) as e:
            F.RgbdBatch(c, imgs, [np.zeros((600, 1000), np.uint16)] * 2, pinned=False).upload()
        assert e.value.code == L.RGBL_E_UNSUPPORTED
        b = F.StereoBatch(c, imgs, imgs, pinned=False)
        b.upload(); b.process_resident(0.5, 175.0)
        assert b.n.min() > 100
    finally:
        c.close()

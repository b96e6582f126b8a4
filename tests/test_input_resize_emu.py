"""The input resize (rgbl_set_input_resize: System::TrackRGBD's / TrackStereo's cv::resize to Settings' new image size) in the whole library
compiled over the CUDA-on-CPU shim (tests/cuda_emu): RGB-D frames (arrays and PNGs) and stereo pairs (arrays and PNGs, alone and together with
rectification) built from input-size images equal, bit for bit, the frames of a context without the resize fed cv2-resized (or remapped)
inputs; every status rule of the setting and of the entry points it changes; after each refused call the context still builds the frames
of a fresh context with the same setting, and clearing the setting gives back the frames of a context that never had it."""
import ctypes as C
import importlib.util
from pathlib import Path

import numpy as np
import pytest

import resize_oracle as RO
from oracle import rectify as RC
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S

HERE = Path(__file__).resolve().parent
W, H, B, NPTS = 160, 120, 4, 400      # context size (Settings::newImSize), max_batch, max_points
SW, SH = 320, 240                     # input size, integer factors (RGB-D and stereo)
TW, TH = 200, 150                     # input size, factor 1.25 (stereo only; the staged-tile kernel form)
N = 2
INV, UNSUP = L.RGBL_E_INVALID, L.RGBL_E_UNSUPPORTED
DEPTH_SCALE, BF, MB, MBF = 0.001, 40.0, 0.4, 40.0
FX, FY, CX, CY = 100.0, 100.0, 80.0, 60.0


@pytest.fixture(scope="module")
def lib():
    spec = importlib.util.spec_from_file_location("cuda_emu_build", HERE / "cuda_emu" / "build.py")
    mod = importlib.util.module_from_spec(spec); spec.loader.exec_module(mod)
    so = C.CDLL(str(mod.build_full()))
    for name, (res, args) in L.SYMBOLS.items():
        fn = getattr(so, name)
        fn.restype, fn.argtypes = res, args
    return so


def _new_ctx(lib, resize=(0, 0)):
    cfg = L.Config(0, W, H, B, NPTS, 0, L.OrbParams(200, 1.2, 4, 20, 7))
    h = C.c_void_p()
    assert lib.rgbl_create(C.byref(cfg), C.byref(h)) == 0
    assert lib.rgbl_set_host_quadtree(h, 1) == 0
    assert lib.rgbl_set_input_resize(h, *resize) == 0
    return h


def cv2_resize(img, w, h):
    try:
        import cv2
        return cv2.resize(img, (w, h), interpolation=cv2.INTER_LINEAR)
    except ImportError:
        return RO.resize_linear(img, w, h)


_KEEP = []


def _ptrs(arrays):
    _KEEP.append(arrays)
    return (C.c_void_p * len(arrays))(*[None if a is None else a.ctypes.data for a in arrays])


def _png(bufs):
    bufs = [np.frombuffer(b, np.uint8) for b in bufs]
    _KEEP.append(bufs)
    return _ptrs(bufs), (C.c_size_t * len(bufs))(*[len(b) for b in bufs])


class Inputs:
    """N frames at input size w x h: images, right images, depth images with holes; their PNG files"""

    def __init__(self, w, h, seed):
        rng = np.random.default_rng(seed)
        self.w, self.h = w, h
        self.img = [S.make_image(seed + f, w, h, 60) for f in range(N)]
        self.right = [np.ascontiguousarray(np.roll(i, -5, axis=1)) for i in self.img]
        self.dep = []
        for _ in range(N):
            d = rng.integers(1000, 20000, (h, w)).astype(np.uint16)
            d[rng.random((h, w)) < 0.2] = 0
            self.dep.append(d)
        self.png = [S.encode_png(i) for i in self.img]
        self.rpng = [S.encode_png(i) for i in self.right]
        self.dpng = [S.encode_png16(d) for d in self.dep]

    def resized(self):
        """the same frames resized on the host to the context's size"""
        r = Inputs.__new__(Inputs)
        r.w, r.h = W, H
        r.img = [cv2_resize(i, W, H) for i in self.img]
        r.right = [cv2_resize(i, W, H) for i in self.right]
        r.dep = [cv2_resize(d, W, H) for d in self.dep]
        return r


BIG, ODD = Inputs(SW, SH, 50), Inputs(TW, TH, 70)


def _download(lib, h, n=N, levels=True):
    cap = lib.rgbl_keypoint_capacity(h)
    kps = np.empty((n, cap), L.KP_DTYPE); desc = np.empty((n, cap, 32), np.uint8)
    dep = np.empty((n, cap), np.float32); ur = np.empty((n, cap), np.float32); cnt = np.zeros(n, np.int32)
    assert lib.rgbl_resident_download(h, L.ptr(kps), L.ptr(desc), L.ptr(dep), L.ptr(ur), cap, L.ptr(cnt)) == 0
    out = [(kps[f, :cnt[f]].tobytes(), desc[f, :cnt[f]].tobytes(), dep[f, :cnt[f]].tobytes(), ur[f, :cnt[f]].tobytes()) for f in range(n)]
    assert cnt.min() > 20
    if levels:                   # level 0 of every frame (stereo: the left frames)
        for f in range(n):
            lvl = np.empty((H, W), np.uint8)
            assert lib.rgbl_orb_get_level(h, f, 0, L.ptr(lvl), W, None, None) == 0
            out.append(lvl.tobytes())
    return out


def _rgbd(lib, h, inp, png=False):
    if png:
        assert lib.rgbl_resident_upload_rgbd_png(h, N, *_png(inp.png), 1, *_png(inp.dpng)) == 0, lib.rgbl_last_error(h)
    else:
        assert lib.rgbl_resident_upload_rgbd(h, N, _ptrs(inp.img), inp.w, inp.h, inp.w, _ptrs(inp.dep), inp.w) == 0, lib.rgbl_last_error(h)
    assert lib.rgbl_resident_process_rgbd(h, DEPTH_SCALE, BF, None) == 0, lib.rgbl_last_error(h)
    return _download(lib, h)


def _stereo(lib, h, inp, png=False):
    if png:
        assert lib.rgbl_resident_upload_stereo_png(h, N, *_png(inp.png), *_png(inp.rpng), 1) == 0, lib.rgbl_last_error(h)
    else:
        assert lib.rgbl_resident_upload_stereo(h, N, _ptrs(inp.img), _ptrs(inp.right), inp.w, inp.h, inp.w) == 0, lib.rgbl_last_error(h)
    assert lib.rgbl_resident_process_stereo(h, MB, MBF, None) == 0, lib.rgbl_last_error(h)
    return _download(lib, h)


@pytest.fixture(scope="module")
def ref(lib):
    """frames of a context without the resize, fed host-resized inputs; and of that context at its own size"""
    h = _new_ctx(lib)
    try:
        out = {"rgbd": _rgbd(lib, h, BIG.resized()), "stereo_big": _stereo(lib, h, BIG.resized()), "stereo_odd": _stereo(lib, h, ODD.resized()),
               "rgbd_own": _rgbd(lib, h, BIG.resized().resized()), "stereo_own": _stereo(lib, h, ODD.resized())}
    finally:
        lib.rgbl_destroy(h)
    return out


def test_rgbd_frames_equal_host_resized_frames(lib, ref):
    h = _new_ctx(lib, (SW, SH))
    try:
        assert _rgbd(lib, h, BIG) == ref["rgbd"]
        assert _rgbd(lib, h, BIG, png=True) == ref["rgbd"]
    finally:
        lib.rgbl_destroy(h)


@pytest.mark.parametrize("inp,key", [(BIG, "stereo_big"), (ODD, "stereo_odd")], ids=["factor2", "factor1.25"])
def test_stereo_frames_equal_host_resized_frames(lib, ref, inp, key):
    h = _new_ctx(lib, (inp.w, inp.h))
    try:
        assert _stereo(lib, h, inp) == ref[key]
        assert _stereo(lib, h, inp, png=True) == ref[key]
    finally:
        lib.rgbl_destroy(h)


def test_resize_with_rectification_is_one_remap(lib):
    """Rectification and resize together: the remap alone reads the input-size images, with maps at the context's size whose
    coordinates index the input-size image (a 1.25 scale with a radial term), as Settings builds them for newImSize."""
    xs, ys = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    r2 = ((xs - W / 2) ** 2 + (ys - H / 2) ** 2) / (W * W)
    mx = np.ascontiguousarray(((xs + 0.5) * TW / W - 0.5) * (1 + 0.05 * r2) - 0.3, np.float32)
    my = np.ascontiguousarray(((ys + 0.5) * TH / H - 0.5) * (1 + 0.05 * r2) + 0.2, np.float32)
    rect = Inputs.__new__(Inputs)
    rect.w, rect.h = W, H
    rect.img = [RC.remap(i, mx, my) for i in ODD.img]
    rect.right = [RC.remap(i, mx, my) for i in ODD.right]
    h0 = _new_ctx(lib)
    try:
        want = _stereo(lib, h0, rect)
    finally:
        lib.rgbl_destroy(h0)
    h = _new_ctx(lib, (TW, TH))
    try:
        assert lib.rgbl_set_stereo_rectification(h, L.ptr(mx), L.ptr(my), L.ptr(mx), L.ptr(my), W) == 0
        assert _stereo(lib, h, ODD) == want
        assert _stereo(lib, h, ODD, png=True) == want
    finally:
        lib.rgbl_destroy(h)


def _rgbl_calls(lib, h):
    """every RGB-L entry point with valid context-size arguments -> statuses"""
    img = [np.zeros((H, W), np.uint8)] * N
    pts = [np.ones((4, 10), np.float32)] * N
    npts = np.full(N, 10, np.int32)
    xyzr = [np.ones((10, 4), np.float32)] * N
    P = np.array([[FX, 0, CX, 0], [0, FY, CY, 0], [0, 0, 1, 0]], np.float32).reshape(12)
    prm = F.make_depth_params(bf=BF)
    cap = lib.rgbl_keypoint_capacity(h)
    kps = np.empty((N, cap), L.KP_DTYPE); desc = np.empty((N, cap, 32), np.uint8); f32 = np.empty((N, cap), np.float32); cnt = np.zeros(N, np.int32)
    io = F.SequenceIO()
    io.n_batches, io.frames_per_batch, io.width, io.height, io.stride = 1, N, W, H, W
    g, p = _ptrs(img), _ptrs(pts)
    io.gray, io.pts4xn, io.n_pts = C.cast(g, C.c_void_p), C.cast(p, C.c_void_p), npts.ctypes.data
    res = [np.zeros((N, 7), np.float32), np.zeros(N, np.int32), np.zeros(N, np.int32)]
    io.poses, io.n_matches, io.n_inliers = (a.ctypes.data for a in res)
    chain = F.make_chain_params([0, 0, 0, 1, 0, 0, 0], FX, FY, CX, CY, BF)
    return [
        lib.rgbl_frame_rgbl_batch(h, N, g, W, H, W, p, L.ptr(npts), L.ptr(P), C.byref(prm), L.ptr(kps), L.ptr(desc), L.ptr(f32), L.ptr(f32), cap, L.ptr(cnt)),
        lib.rgbl_resident_upload(h, N, g, W, H, W, p, L.ptr(npts)),
        lib.rgbl_resident_upload_kitti(h, N, g, W, H, W, _ptrs(xyzr), L.ptr(npts)),
        lib.rgbl_resident_upload_kitti_png(h, N, *_png([S.encode_png(i) for i in img]), 1, _ptrs(xyzr), L.ptr(npts)),
        lib.rgbl_resident_stage(h, 5, N, g, W, H, W, p, L.ptr(npts)),
        lib.rgbl_resident_process(h, L.ptr(P), C.byref(prm), None),
        lib.rgbl_track_sequence(h, L.ptr(P), C.byref(prm), C.byref(chain), C.byref(io)),
    ]


def test_status_rules_keep_the_context_usable(lib, ref):
    h = _new_ctx(lib)
    try:
        # the setting itself: refused values leave the previous setting (off, then SW x SH) in place
        for bad, status in [((-1, SH), INV), ((SW, -1), INV), ((0, SH), INV), ((SW, 0), INV), ((W - 1, SH), UNSUP), ((SW, H - 1), UNSUP)]:
            assert lib.rgbl_set_input_resize(h, *bad) == status, bad
        assert _rgbd(lib, h, BIG.resized().resized()) == ref["rgbd_own"]
        assert lib.rgbl_set_input_resize(h, SW, SH) == 0
        for bad, status in [((-1, SH), INV), ((0, SH), INV), ((W - 1, SH), UNSUP), ((SW, H - 1), UNSUP)]:
            assert lib.rgbl_set_input_resize(h, *bad) == status, bad
            assert _rgbd(lib, h, BIG) == ref["rgbd"]
        # RGB-L is never resized
        assert _rgbl_calls(lib, h) == [UNSUP] * 7
        assert _rgbd(lib, h, BIG) == ref["rgbd"]
        # images or depth images at the context's size (not the input size)
        small = BIG.resized()
        assert lib.rgbl_resident_upload_rgbd(h, N, _ptrs(small.img), W, H, W, _ptrs(small.dep), W) == INV
        assert lib.rgbl_resident_upload_rgbd(h, N, _ptrs(BIG.img), SW, SH, SW, _ptrs(BIG.dep), SW - 1) == INV
        assert lib.rgbl_resident_upload_stereo(h, N, _ptrs(small.img), _ptrs(small.right), W, H, W) == INV
        assert lib.rgbl_resident_upload_rgbd_png(h, N, *_png([S.encode_png(i) for i in small.img]), 1, *_png(BIG.dpng)) == INV
        assert lib.rgbl_resident_upload_rgbd_png(h, N, *_png(BIG.png), 1, *_png([S.encode_png16(d) for d in small.dep])) == INV
        assert _rgbd(lib, h, BIG) == ref["rgbd"]
        # colour image PNGs: the reference resizes before its conversion to gray
        colour = [S.encode_png(S.colorize(i)) for i in BIG.img]
        assert lib.rgbl_resident_upload_rgbd_png(h, N, *_png(colour), 1, *_png(BIG.dpng)) == UNSUP
        assert lib.rgbl_resident_upload_stereo_png(h, N, *_png(colour), *_png(BIG.rpng), 1) == UNSUP
        assert _stereo(lib, h, BIG) == ref["stereo_big"]
        # a factor that is not an integer: stereo only
        assert lib.rgbl_set_input_resize(h, TW, TH) == 0
        assert lib.rgbl_resident_process_stereo(h, MB, MBF, None) == INV             # setting the resize discarded the upload
        assert lib.rgbl_resident_upload_rgbd(h, N, _ptrs(ODD.img), TW, TH, TW, _ptrs(ODD.dep), TW) == UNSUP
        assert lib.rgbl_resident_stage_rgbd(h, 3, N, _ptrs(ODD.img), TW, TH, TW, _ptrs(ODD.dep), TW) == UNSUP
        assert lib.rgbl_resident_upload_rgbd_png(h, N, *_png(ODD.png), 1, *_png(ODD.dpng)) == UNSUP
        assert _stereo(lib, h, ODD) == ref["stereo_odd"]
        # a slot staged at another input size
        assert lib.rgbl_resident_stage_stereo(h, 1, N, _ptrs(ODD.img), _ptrs(ODD.right), TW, TH, TW) == 0
        assert lib.rgbl_set_input_resize(h, SW, SH) == 0
        io = F.SequenceIO()
        io.n_batches, io.frames_per_batch, io.width, io.height, io.stride, io.n_slots, io.first_slot = 1, N, SW, SH, SW, 2, 1
        res = [np.zeros((N, 7), np.float32), np.zeros(N, np.int32), np.zeros(N, np.int32)]
        io.poses, io.n_matches, io.n_inliers = (a.ctypes.data for a in res)
        chain = F.make_chain_params([0, 0, 0, 1, 0, 0, 0], FX, FY, CX, CY, BF)
        assert lib.rgbl_track_sequence_stereo(h, MB, MBF, C.byref(chain), C.byref(io), None) == INV
        assert "another input size" in lib.rgbl_last_error(h).decode()
        assert _stereo(lib, h, BIG) == ref["stereo_big"]
        # a chain in flight
        assert _rgbd(lib, h, BIG, png=True) == ref["rgbd"]
        assert lib.rgbl_resident_track_begin2(h, C.byref(chain)) == 0
        try:
            assert lib.rgbl_set_input_resize(h, 0, 0) == INV
            assert lib.rgbl_set_input_resize(h, TW, TH) == INV
        finally:
            out = [np.zeros((N, 7), np.float32)] + [np.zeros(N, np.int32) for _ in range(4)]
            assert lib.rgbl_resident_track_end2(h, *[L.ptr(a) for a in out]) == 0
        assert _rgbd(lib, h, BIG) == ref["rgbd"]
        # cleared: the frames of a context that never had the setting
        assert lib.rgbl_set_input_resize(h, W, H) == 0
        assert _rgbd(lib, h, BIG.resized().resized()) == ref["rgbd_own"]
        assert lib.rgbl_set_input_resize(h, 0, 0) == 0
        assert _stereo(lib, h, ODD.resized()) == ref["stereo_own"]
    finally:
        lib.rgbl_destroy(h)

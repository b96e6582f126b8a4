"""Colour camera input (rgbl_set_input_channels: the cvtColor of Tracking::GrabImageRGBL / GrabImageRGBD / GrabImageStereo) in the whole
library compiled over the CUDA-on-CPU shim (tests/cuda_emu).  RGB-L, RGB-D and stereo frames built from colour arrays, staged slots and
colour PNGs, with the input resize off / on and (stereo) the rectification off / on, both together included, equal bit for bit the frames
of a gray context fed the images cv2 converts (after cv2's resize or remap of the colour image, as the reference does).  Every status rule
of the setting; after each refused call the context still builds a fresh context's frames, and setting colour then 1 again gives back the
frames of a context that never had the setting."""
import ctypes as C

import numpy as np
import pytest

from test_cuda_emu_colour import BLUE, RED, remap, resize, to_gray
from cuda_emu import build
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S

W, H, B, NPTS = 160, 120, 4, 400      # context size, max_batch, max_points
SW, SH = 320, 240                     # input size of the resize
N = 2
INV, UNSUP = L.RGBL_E_INVALID, L.RGBL_E_UNSUPPORTED
DEPTH_SCALE, BF, MB, MBF = 0.001, 40.0, 0.4, 40.0
FX, FY, CX, CY = 100.0, 100.0, 80.0, 60.0
P = np.array([[FX, 0, CX, 0], [0, FY, CY, 0], [0, 0, 1, 0]], np.float32).reshape(12)


@pytest.fixture(scope="module")
def lib():
    so = C.CDLL(str(build.build_full()))
    for name, (res, args) in L.SYMBOLS.items():
        fn = getattr(so, name)
        fn.restype, fn.argtypes = res, args
    return so


_KEEP = []


def _ptrs(arrays):
    _KEEP.append(arrays)
    return (C.c_void_p * len(arrays))(*[None if a is None else a.ctypes.data for a in arrays])


def _png(bufs):
    bufs = [np.frombuffer(b, np.uint8) for b in bufs]
    _KEEP.append(bufs)
    return _ptrs(bufs), (C.c_size_t * len(bufs))(*[len(b) for b in bufs])


def _maps(sw, sh):
    """context-size maps whose coordinates index sw x sh images (a scale with a radial term), as Settings builds them for newImSize"""
    xs, ys = np.meshgrid(np.arange(W, dtype=np.float64), np.arange(H, dtype=np.float64))
    r2 = ((xs - W / 2) ** 2 + (ys - H / 2) ** 2) / (W * W)
    mx = np.ascontiguousarray(((xs + 0.5) * sw / W - 0.5) * (1 + 0.05 * r2) - 0.3, np.float32)
    my = np.ascontiguousarray(((ys + 0.5) * sh / H - 0.5) * (1 + 0.05 * r2) + 0.2, np.float32)
    return mx, my


class Inputs:
    """N colour frames at w x h (file order R, G, B[, A]), right images, depth images, clouds; their PNG files"""

    def __init__(self, w, h, ch, seed):
        rng = np.random.default_rng(seed)
        self.w, self.h, self.ch = w, h, ch
        gray = [S.make_image(seed + f, w, h, 60) for f in range(N)]
        self.img = [np.ascontiguousarray(S.colorize(g, seed + f, alpha=ch == 4)) for f, g in enumerate(gray)]
        self.right = [np.ascontiguousarray(np.roll(i, -5, axis=1)) for i in self.img]
        self.dep = []
        for _ in range(N):
            d = rng.integers(1000, 20000, (h, w)).astype(np.uint16)
            d[rng.random((h, w)) < 0.2] = 0
            self.dep.append(d)
        self.png = [S.encode_png(i) for i in self.img]
        self.rpng = [S.encode_png(i) for i in self.right]
        self.dpng = [S.encode_png16(d) for d in self.dep]

    def gray(self, w0, size=None, maps=None):
        """what a gray context is fed: the colour images remapped (maps) or resized (size), then converted with channel 0 weighted w0"""
        def f(i):
            if maps is not None:
                i = remap(i, *maps)
            elif size is not None:
                i = resize(i, *size)
            return to_gray(i, w0)
        g = Inputs.__new__(Inputs)
        g.ch = 1
        g.img, g.right = [f(i) for i in self.img], [f(i) for i in self.right]
        g.h, g.w = g.img[0].shape
        g.dep = [resize(d, *size) for d in self.dep] if size is not None else self.dep
        return g


CLOUDS = [np.ascontiguousarray(S.make_pointcloud(f, n_azimuth=60)[:, :NPTS]) for f in range(N)]
BIG3, BIG4, SMALL3 = Inputs(SW, SH, 3, 50), Inputs(SW, SH, 4, 60), Inputs(W, H, 3, 70)


def _new_ctx(lib, channels=1, camera_rgb=1, resize_to=(0, 0), maps=None):
    cfg = L.Config(0, W, H, B, NPTS, 0, L.OrbParams(200, 1.2, 4, 20, 7))
    h = C.c_void_p()
    assert lib.rgbl_create(C.byref(cfg), C.byref(h)) == 0
    assert lib.rgbl_set_host_quadtree(h, 1) == 0
    assert lib.rgbl_set_input_resize(h, *resize_to) == 0
    assert lib.rgbl_set_input_channels(h, channels, camera_rgb) == 0
    if maps is not None:
        assert lib.rgbl_set_stereo_rectification(h, L.ptr(maps[0]), L.ptr(maps[1]), L.ptr(maps[0]), L.ptr(maps[1]), W) == 0
    return h


def _download(lib, h, n=N):
    cap = lib.rgbl_keypoint_capacity(h)
    kps = np.empty((n, cap), L.KP_DTYPE); desc = np.empty((n, cap, 32), np.uint8)
    dep = np.empty((n, cap), np.float32); ur = np.empty((n, cap), np.float32); cnt = np.zeros(n, np.int32)
    assert lib.rgbl_resident_download(h, L.ptr(kps), L.ptr(desc), L.ptr(dep), L.ptr(ur), cap, L.ptr(cnt)) == 0
    out = [(kps[f, :cnt[f]].tobytes(), desc[f, :cnt[f]].tobytes(), dep[f, :cnt[f]].tobytes(), ur[f, :cnt[f]].tobytes()) for f in range(n)]
    assert cnt.min() > 10
    for f in range(n):
        lvl = np.empty((H, W), np.uint8)
        assert lib.rgbl_orb_get_level(h, f, 0, L.ptr(lvl), W, None, None) == 0
        out.append(lvl.tobytes())
    return out


def _stride(inp):
    return inp.w * inp.ch


def _rgbl(lib, h, inp, png=False, camera_rgb=1):
    pts, npts = _ptrs(CLOUDS), np.array([c.shape[1] for c in CLOUDS], np.int32)
    if png:
        xyzr = [np.ascontiguousarray(c.T) for c in CLOUDS]
        assert lib.rgbl_resident_upload_kitti_png(h, N, *_png(inp.png), camera_rgb, _ptrs(xyzr), L.ptr(npts)) == 0, lib.rgbl_last_error(h)
    else:
        assert lib.rgbl_resident_upload(h, N, _ptrs(inp.img), inp.w, inp.h, _stride(inp), pts, L.ptr(npts)) == 0, lib.rgbl_last_error(h)
    assert lib.rgbl_resident_process(h, L.ptr(P), C.byref(F.make_depth_params(bf=BF)), None) == 0, lib.rgbl_last_error(h)
    return _download(lib, h)


def _rgbd(lib, h, inp, png=False, camera_rgb=1):
    if png:
        assert lib.rgbl_resident_upload_rgbd_png(h, N, *_png(inp.png), camera_rgb, *_png(inp.dpng)) == 0, lib.rgbl_last_error(h)
    else:
        assert lib.rgbl_resident_upload_rgbd(h, N, _ptrs(inp.img), inp.w, inp.h, _stride(inp), _ptrs(inp.dep), inp.w) == 0, lib.rgbl_last_error(h)
    assert lib.rgbl_resident_process_rgbd(h, DEPTH_SCALE, BF, None) == 0, lib.rgbl_last_error(h)
    return _download(lib, h)


def _stereo(lib, h, inp, png=False, camera_rgb=1):
    if png:
        assert lib.rgbl_resident_upload_stereo_png(h, N, *_png(inp.png), *_png(inp.rpng), camera_rgb) == 0, lib.rgbl_last_error(h)
    else:
        assert lib.rgbl_resident_upload_stereo(h, N, _ptrs(inp.img), _ptrs(inp.right), inp.w, inp.h, _stride(inp)) == 0, lib.rgbl_last_error(h)
    assert lib.rgbl_resident_process_stereo(h, MB, MBF, None) == 0, lib.rgbl_last_error(h)
    return _download(lib, h)


def _gray(lib, run, inp):
    h = _new_ctx(lib)
    try:
        return run(lib, h, inp)
    finally:
        lib.rgbl_destroy(h)


# a PNG file holds R, G, B: imread's B, G, R order with Camera.RGB = 1 weights the file's channel 0 (red) as blue
PNG_W0 = {1: BLUE, 0: RED}


@pytest.mark.parametrize("camera_rgb", [1, 0])
@pytest.mark.parametrize("inp", [SMALL3, Inputs(W, H, 4, 80)], ids=["rgb", "rgba"])
def test_rgbl_frames_equal_host_converted_frames(lib, inp, camera_rgb):
    h = _new_ctx(lib, inp.ch, camera_rgb)
    try:
        assert _rgbl(lib, h, inp) == _gray(lib, _rgbl, inp.gray(RED if camera_rgb else BLUE))
        assert _rgbl(lib, h, inp, png=True, camera_rgb=camera_rgb) == _gray(lib, _rgbl, inp.gray(PNG_W0[camera_rgb]))
    finally:
        lib.rgbl_destroy(h)


@pytest.mark.parametrize("resized", [False, True], ids=["own_size", "resize"])
def test_rgbd_frames_equal_host_converted_frames(lib, resized):
    inp = BIG4 if resized else SMALL3
    h = _new_ctx(lib, inp.ch, 1, (SW, SH) if resized else (0, 0))
    size = (W, H) if resized else None
    try:
        assert _rgbd(lib, h, inp) == _gray(lib, _rgbd, inp.gray(RED, size))
        assert _rgbd(lib, h, inp, png=True, camera_rgb=0) == _gray(lib, _rgbd, inp.gray(PNG_W0[0], size))
    finally:
        lib.rgbl_destroy(h)


STEREO = [("own_size", SMALL3, (0, 0), None), ("resize", BIG3, (SW, SH), None), ("rectify", SMALL3, (0, 0), _maps(W, H)),
          ("resize_rectify", BIG4, (SW, SH), _maps(SW, SH))]


@pytest.mark.parametrize("name,inp,resize_to,maps", STEREO, ids=[s[0] for s in STEREO])
def test_stereo_frames_equal_host_converted_frames(lib, name, inp, resize_to, maps):
    h = _new_ctx(lib, inp.ch, 1, resize_to, maps)
    size = (W, H) if resize_to != (0, 0) else None
    try:
        assert _stereo(lib, h, inp) == _gray(lib, _stereo, inp.gray(RED, size, maps))
        assert _stereo(lib, h, inp, png=True, camera_rgb=1) == _gray(lib, _stereo, inp.gray(PNG_W0[1], size, maps))
    finally:
        lib.rgbl_destroy(h)


def test_gray_png_on_a_colour_context_with_a_raw_stage(lib):
    """a colour context also takes gray PNG streams: with the resize on they are resized as gray planes"""
    g = BIG3.gray(RED)
    g.png, g.rpng = [S.encode_png(i) for i in g.img], [S.encode_png(i) for i in g.right]
    h = _new_ctx(lib, 3, 1, (SW, SH))
    try:
        h0 = _new_ctx(lib, 1, 1, (SW, SH))
        try:
            want = _stereo(lib, h0, g, png=True)
        finally:
            lib.rgbl_destroy(h0)
        assert _stereo(lib, h, g, png=True) == want
    finally:
        lib.rgbl_destroy(h)


def _io(inp, n_slots=0):
    io = F.SequenceIO()
    io.n_batches, io.frames_per_batch, io.width, io.height, io.stride = 1, N, inp.w, inp.h, _stride(inp)
    io.n_slots, io.first_slot = n_slots, 0
    res = [np.zeros((N, 7), np.float32), np.zeros(N, np.int32), np.zeros(N, np.int32)]
    _KEEP.append(res)
    io.poses, io.n_matches, io.n_inliers = (a.ctypes.data for a in res)
    if not n_slots:
        io.gray = C.cast(_ptrs(inp.img), C.c_void_p)
    return io, res


CHAIN = F.make_chain_params([0, 0, 0, 1, 0, 0, 0], FX, FY, CX, CY, BF, th_last=7.0, th_local=1.0)


def _stereo_runner(lib, h, inp, resident):
    if resident:
        assert lib.rgbl_resident_stage_stereo(h, 0, N, _ptrs(inp.img), _ptrs(inp.right), inp.w, inp.h, _stride(inp)) == 0, lib.rgbl_last_error(h)
    io, res = _io(inp, 1 if resident else 0)
    assert lib.rgbl_track_sequence_stereo(h, MB, MBF, C.byref(CHAIN), C.byref(io), None if resident else _ptrs(inp.right)) == 0, lib.rgbl_last_error(h)
    return [r.tobytes() for r in res]


@pytest.mark.parametrize("resident", [False, True], ids=["host", "staged"])
def test_stereo_runner_equals_host_converted_runner(lib, resident):
    h = _new_ctx(lib, 3, 1)
    try:
        assert _stereo_runner(lib, h, SMALL3, resident) == _gray(lib, lambda l, c, i: _stereo_runner(l, c, i, resident), SMALL3.gray(RED))
    finally:
        lib.rgbl_destroy(h)


def test_status_rules_keep_the_context_usable(lib):
    g = SMALL3.gray(RED)
    ref3 = ref_own = _gray(lib, _stereo, g)         # the colour pairs on a colour context, their gray images on a gray one
    h = _new_ctx(lib)
    try:
        # refused values leave the previous setting (gray, then 3 channels RGB) in place
        for bad in [(0, 1), (2, 1), (5, 1), (-1, 0), (3, 2), (3, -1), (1, 7)]:
            assert lib.rgbl_set_input_channels(h, *bad) == INV, bad
        assert _stereo(lib, h, g) == ref_own
        assert lib.rgbl_set_input_channels(h, 3, 1) == 0
        for bad in [(0, 1), (2, 0), (4, 2)]:
            assert lib.rgbl_set_input_channels(h, *bad) == INV, bad
            assert _stereo(lib, h, SMALL3) == ref3
        # a row stride below width * channels
        assert lib.rgbl_resident_upload_stereo(h, N, _ptrs(SMALL3.img), _ptrs(SMALL3.right), W, H, 3 * W - 1) == INV
        assert lib.rgbl_resident_stage_stereo(h, 2, N, _ptrs(SMALL3.img), _ptrs(SMALL3.right), W, H, W) == INV
        assert _stereo(lib, h, SMALL3) == ref3
        # setting (or clearing) the value discards a pending upload
        assert lib.rgbl_resident_upload_stereo(h, N, _ptrs(SMALL3.img), _ptrs(SMALL3.right), W, H, 3 * W) == 0
        assert lib.rgbl_set_input_channels(h, 3, 1) == 0
        assert lib.rgbl_resident_process_stereo(h, MB, MBF, None) == INV
        assert _stereo(lib, h, SMALL3) == ref3
        # a slot staged with another channel count
        assert lib.rgbl_resident_stage_stereo(h, 1, N, _ptrs(SMALL3.img), _ptrs(SMALL3.right), W, H, 3 * W) == 0
        assert lib.rgbl_set_input_channels(h, 4, 1) == 0
        io, _ = _io(SMALL3, 2)
        io.first_slot = 1
        assert lib.rgbl_track_sequence_stereo(h, MB, MBF, C.byref(CHAIN), C.byref(io), None) == INV
        assert "another channel count" in lib.rgbl_last_error(h).decode()
        assert lib.rgbl_set_input_channels(h, 3, 1) == 0
        assert _stereo(lib, h, SMALL3) == ref3
        # a chain in flight
        assert lib.rgbl_resident_track_begin2(h, C.byref(CHAIN)) == 0
        try:
            assert lib.rgbl_set_input_channels(h, 1, 1) == INV
            assert lib.rgbl_set_input_channels(h, 4, 0) == INV
        finally:
            out = [np.zeros((N, 7), np.float32)] + [np.zeros(N, np.int32) for _ in range(4)]
            assert lib.rgbl_resident_track_end2(h, *[L.ptr(a) for a in out]) == 0
        assert _stereo(lib, h, SMALL3) == ref3
        # the calls that keep taking 8-bit gray images on a colour context
        pts, npts = _ptrs(CLOUDS), np.array([c.shape[1] for c in CLOUDS], np.int32)
        cap = lib.rgbl_keypoint_capacity(h)
        kps = np.empty((N, cap), L.KP_DTYPE); desc = np.empty((N, cap, 32), np.uint8); f32 = np.empty((N, cap), np.float32); cnt = np.zeros(N, np.int32)
        assert lib.rgbl_frame_rgbl_batch(h, N, _ptrs(g.img), W, H, W, pts, L.ptr(npts), L.ptr(P), C.byref(F.make_depth_params(bf=BF)), L.ptr(kps),
                                         L.ptr(desc), L.ptr(f32), L.ptr(f32), cap, L.ptr(cnt)) == 0
        assert _rgbl(lib, h, SMALL3) == _gray(lib, _rgbl, g)
        # back to 1: the frames of a context that never had the setting
        assert lib.rgbl_set_input_channels(h, 1, 0) == 0
        assert _stereo(lib, h, g) == ref_own
    finally:
        lib.rgbl_destroy(h)


def test_gray_context_refuses_colour_pngs_with_a_raw_stage(lib):
    h = _new_ctx(lib, 1, 1, (SW, SH))
    try:
        assert lib.rgbl_resident_upload_stereo_png(h, N, *_png(BIG3.png), *_png(BIG3.rpng), 1) == UNSUP
        assert lib.rgbl_set_input_channels(h, 3, 1) == 0
        assert _stereo(lib, h, BIG3, png=True) == _gray(lib, _stereo, BIG3.gray(PNG_W0[1], (W, H)))
    finally:
        lib.rgbl_destroy(h)

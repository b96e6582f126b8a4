"""Input paths of frame construction: every upload, PNG upload, stage, process and sequence-runner entry point of each input kind
(RGB-L, RGB-D, stereo) called with inputs that have one fault each, against the whole library compiled over the CUDA-on-CPU shim
(tests/cuda_emu).  Each case asserts its status code.  After each refused call the same context must still build frames: one valid
batch of the case's kind is uploaded, processed and downloaded, and must equal a fresh context's outputs bit for bit.  Every runner
case is refused before its tracking chain starts."""
import ctypes as C

import numpy as np
import pytest

from cuda_emu import build
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S

W, H, B, NPTS = 160, 120, 4, 400      # context size, max_batch, max_points
N = 2                                 # frames (RGB-L, RGB-D) or pairs (stereo) of a valid batch
INV, CAP, EMPTY, UNSUP = L.RGBL_E_INVALID, L.RGBL_E_CAPACITY, L.RGBL_E_EMPTY, L.RGBL_E_UNSUPPORTED
DEPTH_SCALE, BF, MB, MBF = 0.001, 40.0, 0.4, 40.0
FX, FY, CX, CY = 100.0, 100.0, 80.0, 60.0


@pytest.fixture(scope="module")
def lib():
    so = C.CDLL(str(build.build_full()))
    for name, (res, args) in L.SYMBOLS.items():
        fn = getattr(so, name)
        fn.restype, fn.argtypes = res, args
    return so


def _new_ctx(lib, max_points=NPTS):
    cfg = L.Config(0, W, H, B, max_points, 0, L.OrbParams(200, 1.2, 4, 20, 7))
    h = C.c_void_p()
    assert lib.rgbl_create(C.byref(cfg), C.byref(h)) == 0
    assert lib.rgbl_set_host_quadtree(h, 1) == 0          # the quicker of the two quad-trees under emulation
    return h


_KEEP = []          # arrays whose addresses were handed out: kept alive for the module's lifetime


def _ptrs(arrays):
    _KEEP.append(arrays)
    return (C.c_void_p * len(arrays))(*[None if a is None else a.ctypes.data for a in arrays])


def _sizes(bufs):
    return (C.c_size_t * len(bufs))(*[len(b) for b in bufs])


class Inputs:
    """B frames of each input: images, planar clouds in the camera frame (P = K [I | 0]), KITTI .bin records, depth images, right
    images, and the PNG files of images and depth images."""

    def __init__(self):
        rng = np.random.default_rng(7)
        self.img = [S.make_image(30 + f, W, H, 40) for f in range(B)]
        self.right = [np.ascontiguousarray(np.roll(i, -3, axis=1)) for i in self.img]
        self.clouds, self.xyzr = [], []
        for f in range(B):
            n = 300 + 20 * f
            z = rng.uniform(6.0, 40.0, n)
            x = (rng.uniform(0, W, n) - CX) * z / FX; y = (rng.uniform(0, H, n) - CY) * z / FY
            self.clouds.append(np.ascontiguousarray(np.stack([x, y, z, np.ones(n)]).astype(np.float32)))
            self.xyzr.append(np.ascontiguousarray(np.stack([x, y, z, rng.uniform(0, 1, n)], 1).astype(np.float32)))
        self.npts = np.array([c.shape[1] for c in self.clouds], np.int32)
        self.dep = [rng.integers(1000, 20000, (H, W)).astype(np.uint16) for _ in range(B)]
        self.png = [S.encode_png(i) for i in self.img]
        self.rpng = [S.encode_png(i) for i in self.right]
        self.dpng = [S.encode_png16(d) for d in self.dep]
        self.P = np.array([[FX, 0, CX, 0], [0, FY, CY, 0], [0, 0, 1, 0]], np.float32).reshape(12)
        self.prm = L.DepthParams()
        self.prm.method, self.prm.min_dist, self.prm.max_dist, self.prm.bf, self.prm.inv_dilation_scale = L.DEPTH_INVERSE_DILATION, 5.0, 200.0, BF, 1.0
        self.prm.ku = self.prm.kv = 5
        flat = np.zeros(81, np.uint8); flat[:25] = S.structuring_element("diamond", 5).reshape(-1)
        C.memmove(self.prm.mask, flat.ctypes.data, 81)
        self.prm.avg_kernel, self.prm.nn_search_radius = 5, 7.0

    def g(self, n=N, null=None):
        return _ptrs([None if f == null else self.img[f] for f in range(n)])

    def r(self, n=N, null=None):
        return _ptrs([None if f == null else self.right[f] for f in range(n)])

    def pts(self, n=N, null=None):
        return _ptrs([None if f == null else self.clouds[f] for f in range(n)])

    def kitti(self, n=N):
        return _ptrs(self.xyzr[:n])

    def n_pts(self, n=N, f=None, value=None):
        a = np.ascontiguousarray(self.npts[:n].copy())
        if f is not None:
            a[f] = value
        return a

    def d(self, n=N, null=None):
        return _ptrs([None if f == null else self.dep[f] for f in range(n)])

    def pngs(self, which="png", n=N, empty=None, small=None):
        bufs = [np.frombuffer(b, np.uint8) for b in getattr(self, which)[:n]]
        if small is not None:
            bufs[small] = np.frombuffer(S.encode_png(self.img[small][:-2, :-4]) if which != "dpng" else S.encode_png16(self.dep[small][:-2, :-4]), np.uint8)
        sizes = [0 if f == empty else len(b) for f, b in enumerate(bufs)]
        return _ptrs(bufs), (C.c_size_t * n)(*sizes), bufs


IN = Inputs()


def _download(lib, h, n):
    cap = lib.rgbl_keypoint_capacity(h)
    kps = np.empty((n, cap), L.KP_DTYPE); desc = np.empty((n, cap, 32), np.uint8)
    dep = np.empty((n, cap), np.float32); ur = np.empty((n, cap), np.float32); cnt = np.zeros(n, np.int32)
    assert lib.rgbl_resident_download(h, L.ptr(kps), L.ptr(desc), L.ptr(dep), L.ptr(ur), cap, L.ptr(cnt)) == 0
    return [(kps[f, :cnt[f]].tobytes(), desc[f, :cnt[f]].tobytes(), dep[f, :cnt[f]].tobytes(), ur[f, :cnt[f]].tobytes()) for f in range(n)]


def _build(lib, h, kind):
    """Upload, process and download one valid batch of `kind` -> bytes of every output."""
    cnt = np.zeros(N, np.int32)
    if kind == "rgbl":
        assert lib.rgbl_resident_upload(h, N, IN.g(), W, H, W, IN.pts(), L.ptr(IN.n_pts())) == 0
        assert lib.rgbl_resident_process(h, L.ptr(IN.P), C.byref(IN.prm), L.ptr(cnt)) == 0
    elif kind == "rgbd":
        assert lib.rgbl_resident_upload_rgbd(h, N, IN.g(), W, H, W, IN.d(), W) == 0
        assert lib.rgbl_resident_process_rgbd(h, DEPTH_SCALE, BF, L.ptr(cnt)) == 0
    else:
        assert lib.rgbl_resident_upload_stereo(h, N, IN.g(), IN.r(), W, H, W) == 0
        assert lib.rgbl_resident_process_stereo(h, MB, MBF, L.ptr(cnt)) == 0
    out = _download(lib, h, N)
    assert [len(o[0]) // L.KP_DTYPE.itemsize for o in out] == cnt.tolist() and cnt.min() > 20
    return out


def _seq_io(T=N, n_batches=1, gray=None, pts=None, n_pts=None, n_slots=0, first_slot=0, width=W, stride=W):
    io = F.SequenceIO()
    io.n_batches, io.frames_per_batch, io.width, io.height, io.stride = n_batches, T, width, H, stride
    io.gray = None if gray is None else C.cast(gray, C.c_void_p)
    io.pts4xn = None if pts is None else C.cast(pts, C.c_void_p)
    io.n_pts = None if n_pts is None else n_pts.ctypes.data
    io.n_slots, io.first_slot = n_slots, first_slot
    io._keep = [gray, pts, n_pts, np.zeros((T * n_batches, 7), np.float32), np.zeros(T * n_batches, np.int32), np.zeros(T * n_batches, np.int32)]
    io.poses, io.n_matches, io.n_inliers = (a.ctypes.data for a in io._keep[3:])
    return io


CHAIN = F.make_chain_params([0, 0, 0, 1, 0, 0, 0], FX, FY, CX, CY, BF)
# staged slots of the shared context (staged once, before the cases run): 0 RGB-L, 1 RGB-D, 2 stereo, each with N frames / pairs;
# slot 7 is never staged
SLOT_RGBL, SLOT_RGBD, SLOT_STEREO, SLOT_EMPTY = 0, 1, 2, 7


def _rgbl(lib, h, io, P=IN.P, prm=IN.prm):
    return lib.rgbl_track_sequence(h, None if P is None else L.ptr(P), None if prm is None else C.byref(prm), C.byref(CHAIN), C.byref(io))


def _rgbd(lib, h, io, depth=None, depth_stride=W, depth_scale=DEPTH_SCALE, bf=BF):
    return lib.rgbl_track_sequence_rgbd(h, depth_scale, bf, C.byref(CHAIN), C.byref(io), depth, depth_stride)


def _stereo(lib, h, io, right=None, mb=MB, mbf=MBF):
    return lib.rgbl_track_sequence_stereo(h, mb, mbf, C.byref(CHAIN), C.byref(io), right)


def _distorted(call):
    """`call` with a distorted camera (k1 != 0), then the undistorted camera again."""
    def run(lib, h):
        dist = np.array([-0.1, 0.01, 0.0, 0.0], np.float32)
        assert lib.rgbl_set_camera_distortion(h, FX, FY, CX, CY, L.ptr(dist), 4, None) == 0
        try:
            return call(lib, h)
        finally:
            assert lib.rgbl_set_camera_distortion(h, FX, FY, CX, CY, L.ptr(np.zeros(4, np.float32)), 4, None) == 0
    return run


def _after(kind, call):
    """`call` after a valid upload of `kind`."""
    def run(lib, h):
        if kind == "rgbl":
            assert lib.rgbl_resident_upload(h, N, IN.g(), W, H, W, IN.pts(), L.ptr(IN.n_pts())) == 0
        elif kind == "rgbd":
            assert lib.rgbl_resident_upload_rgbd(h, N, IN.g(), W, H, W, IN.d(), W) == 0
        else:
            assert lib.rgbl_resident_upload_stereo(h, N, IN.g(), IN.r(), W, H, W) == 0
        return call(lib, h)
    return run


def _frame_rgbl(lib, h, n=N, gray=None, pts=None, n_pts=None, width=W, stride=W, P=IN.P, prm=IN.prm):
    cap = lib.rgbl_keypoint_capacity(h)
    kps = np.empty((max(n, 1), cap), L.KP_DTYPE); desc = np.empty((max(n, 1), cap, 32), np.uint8)
    dep = np.empty((max(n, 1), cap), np.float32); ur = np.empty((max(n, 1), cap), np.float32); cnt = np.zeros(max(n, 1), np.int32)
    gray = IN.g(max(n, 1)) if gray is None else gray
    pts = IN.pts(max(n, 1)) if pts is None else pts
    n_pts = IN.n_pts(max(n, 1)) if n_pts is None else n_pts
    return lib.rgbl_frame_rgbl_batch(h, n, gray, width, H, stride, pts, L.ptr(n_pts) if isinstance(n_pts, np.ndarray) else n_pts,
                                     None if P is None else L.ptr(P), None if prm is None else C.byref(prm),
                                     L.ptr(kps), L.ptr(desc), L.ptr(dep), L.ptr(ur), cap, L.ptr(cnt))


def _prm(**kw):
    p = L.DepthParams()
    C.memmove(C.byref(p), C.byref(IN.prm), C.sizeof(p))
    for k, v in kw.items():
        setattr(p, k, v)
    return p


def _png_args(which="png", n=N, empty=None, small=None):
    p, s, _ = IN.pngs(which, n, empty, small)
    return p, s


# (id, kind of the valid batch built afterwards, expected status, call(lib, h))
CASES = [
    # ---- RGB-L: rgbl_frame_rgbl_batch ----
    ("frame_rgbl/null_gray", "rgbl", INV, lambda lib, h: lib.rgbl_frame_rgbl_batch(h, N, None, W, H, W, IN.pts(), L.ptr(IN.n_pts()), L.ptr(IN.P), C.byref(IN.prm), None, None, None, None, 0, None)),
    ("frame_rgbl/null_clouds", "rgbl", INV, lambda lib, h: _frame_rgbl(lib, h, pts=C.c_void_p())),
    ("frame_rgbl/null_prm", "rgbl", INV, lambda lib, h: _frame_rgbl(lib, h, prm=None)),
    ("frame_rgbl/empty_image", "rgbl", EMPTY, lambda lib, h: _frame_rgbl(lib, h, gray=IN.g(null=1))),
    ("frame_rgbl/zero_width", "rgbl", EMPTY, lambda lib, h: _frame_rgbl(lib, h, width=0)),
    ("frame_rgbl/wrong_width", "rgbl", INV, lambda lib, h: _frame_rgbl(lib, h, width=W - 2, stride=W)),
    ("frame_rgbl/stride_below_width", "rgbl", INV, lambda lib, h: _frame_rgbl(lib, h, stride=W - 1)),
    ("frame_rgbl/zero_frames", "rgbl", INV, lambda lib, h: _frame_rgbl(lib, h, n=0)),
    ("frame_rgbl/frames_above_max_batch", "rgbl", CAP, lambda lib, h: _frame_rgbl(lib, h, n=B + 1, gray=_ptrs(IN.img + [IN.img[0]]), pts=_ptrs(IN.clouds + [IN.clouds[0]]), n_pts=np.append(IN.npts, IN.npts[0]).astype(np.int32))),
    ("frame_rgbl/cloud_above_max_points", "rgbl", CAP, lambda lib, h: _frame_rgbl(lib, h, n_pts=IN.n_pts(f=1, value=NPTS + 1))),
    ("frame_rgbl/negative_cloud_size", "rgbl", CAP, lambda lib, h: _frame_rgbl(lib, h, n_pts=IN.n_pts(f=0, value=-1))),
    ("frame_rgbl/null_cloud", "rgbl", CAP, lambda lib, h: _frame_rgbl(lib, h, pts=IN.pts(null=1))),
    ("frame_rgbl/empty_image_and_bad_cloud", "rgbl", CAP, lambda lib, h: _frame_rgbl(lib, h, gray=IN.g(null=1), n_pts=IN.n_pts(f=0, value=NPTS + 1))),
    ("frame_rgbl/bad_cloud_after_empty_image", "rgbl", EMPTY, lambda lib, h: _frame_rgbl(lib, h, gray=IN.g(null=0), n_pts=IN.n_pts(f=1, value=NPTS + 1))),
    ("frame_rgbl/structuring_element_10", "rgbl", INV, lambda lib, h: _frame_rgbl(lib, h, prm=_prm(ku=10))),
    ("frame_rgbl/unknown_depth_method", "rgbl", UNSUP, lambda lib, h: _frame_rgbl(lib, h, prm=_prm(method=7))),
    # ---- RGB-L: uploads ----
    ("upload/null_gray", "rgbl", INV, lambda lib, h: lib.rgbl_resident_upload(h, N, None, W, H, W, IN.pts(), L.ptr(IN.n_pts()))),
    ("upload/null_counts", "rgbl", INV, lambda lib, h: lib.rgbl_resident_upload(h, N, IN.g(), W, H, W, IN.pts(), None)),
    ("upload/empty_image", "rgbl", EMPTY, lambda lib, h: lib.rgbl_resident_upload(h, N, IN.g(null=0), W, H, W, IN.pts(), L.ptr(IN.n_pts()))),
    ("upload/wrong_height", "rgbl", INV, lambda lib, h: lib.rgbl_resident_upload(h, N, IN.g(), W, H - 1, W, IN.pts(), L.ptr(IN.n_pts()))),
    ("upload/frames_above_max_batch", "rgbl", CAP, lambda lib, h: lib.rgbl_resident_upload(h, B + 1, _ptrs(IN.img + [IN.img[0]]), W, H, W, _ptrs(IN.clouds + [IN.clouds[0]]), L.ptr(np.append(IN.npts, 1).astype(np.int32)))),
    ("upload/cloud_above_max_points", "rgbl", CAP, lambda lib, h: lib.rgbl_resident_upload(h, N, IN.g(), W, H, W, IN.pts(), L.ptr(IN.n_pts(f=1, value=NPTS + 1)))),
    ("upload_kitti/null_records", "rgbl", INV, lambda lib, h: lib.rgbl_resident_upload_kitti(h, N, IN.g(), W, H, W, None, L.ptr(IN.n_pts()))),
    ("upload_kitti/empty_image", "rgbl", EMPTY, lambda lib, h: lib.rgbl_resident_upload_kitti(h, N, IN.g(null=1), W, H, W, IN.kitti(), L.ptr(IN.n_pts()))),
    ("upload_kitti/stride_below_width", "rgbl", INV, lambda lib, h: lib.rgbl_resident_upload_kitti(h, N, IN.g(), W, H, W - 1, IN.kitti(), L.ptr(IN.n_pts()))),
    ("upload_kitti/cloud_above_max_points", "rgbl", CAP, lambda lib, h: lib.rgbl_resident_upload_kitti(h, N, IN.g(), W, H, W, IN.kitti(), L.ptr(IN.n_pts(f=0, value=NPTS + 1)))),
    ("upload_kitti_png/null_png", "rgbl", INV, lambda lib, h: lib.rgbl_resident_upload_kitti_png(h, N, None, None, 1, IN.kitti(), L.ptr(IN.n_pts()))),
    ("upload_kitti_png/empty_stream", "rgbl", EMPTY, lambda lib, h: lib.rgbl_resident_upload_kitti_png(h, N, *_png_args(empty=1), 1, IN.kitti(), L.ptr(IN.n_pts()))),
    ("upload_kitti_png/wrong_size", "rgbl", INV, lambda lib, h: lib.rgbl_resident_upload_kitti_png(h, N, *_png_args(small=0), 1, IN.kitti(), L.ptr(IN.n_pts()))),
    ("upload_kitti_png/frames_above_max_batch", "rgbl", CAP, lambda lib, h: lib.rgbl_resident_upload_kitti_png(h, B + 1, *_png_args(n=B), 1, IN.kitti(B), L.ptr(IN.n_pts(B)))),
    ("upload_kitti_png/cloud_above_max_points", "rgbl", CAP, lambda lib, h: lib.rgbl_resident_upload_kitti_png(h, N, *_png_args(), 1, IN.kitti(), L.ptr(IN.n_pts(f=1, value=NPTS + 1)))),
    ("decode_png_gray/null_output", "rgbl", INV, lambda lib, h: lib.rgbl_decode_png_gray(h, N, *_png_args(), 1, _ptrs([np.empty((H, W), np.uint8), None]), W)),
    ("decode_png_gray/empty_stream", "rgbl", EMPTY, lambda lib, h: lib.rgbl_decode_png_gray(h, N, *_png_args(empty=0), 1, _ptrs([np.empty((H, W), np.uint8)] * N), W)),
    # ---- RGB-L: process ----
    ("process/after_rgbd_upload", "rgbl", INV, _after("rgbd", lambda lib, h: lib.rgbl_resident_process(h, L.ptr(IN.P), C.byref(IN.prm), None))),
    ("process/after_stereo_upload", "rgbl", INV, _after("stereo", lambda lib, h: lib.rgbl_resident_process(h, L.ptr(IN.P), C.byref(IN.prm), None))),
    ("process/null_P", "rgbl", INV, _after("rgbl", lambda lib, h: lib.rgbl_resident_process(h, None, C.byref(IN.prm), None))),
    ("process/average_kernel_10", "rgbl", INV, _after("rgbl", lambda lib, h: lib.rgbl_resident_process(h, L.ptr(IN.P), C.byref(_prm(method=L.DEPTH_AVERAGE_FILTERING, avg_kernel=10)), None))),
    ("process/nn_radius_31", "rgbl", INV, _after("rgbl", lambda lib, h: lib.rgbl_resident_process(h, L.ptr(IN.P), C.byref(_prm(method=L.DEPTH_NEAREST_NEIGHBOR_PIXEL, nn_search_radius=31.0)), None))),
    # ---- RGB-L: stage ----
    ("stage/slot_below_range", "rgbl", INV, lambda lib, h: lib.rgbl_resident_stage(h, -1, N, IN.g(), W, H, W, IN.pts(), L.ptr(IN.n_pts()))),
    ("stage/slot_above_range", "rgbl", INV, lambda lib, h: lib.rgbl_resident_stage(h, 8, N, IN.g(), W, H, W, IN.pts(), L.ptr(IN.n_pts()))),
    ("stage/null_clouds", "rgbl", INV, lambda lib, h: lib.rgbl_resident_stage(h, 3, N, IN.g(), W, H, W, None, L.ptr(IN.n_pts()))),
    ("stage/empty_image", "rgbl", EMPTY, lambda lib, h: lib.rgbl_resident_stage(h, 3, N, IN.g(null=1), W, H, W, IN.pts(), L.ptr(IN.n_pts()))),
    ("stage/wrong_width", "rgbl", INV, lambda lib, h: lib.rgbl_resident_stage(h, 3, N, IN.g(), W + 1, H, W + 1, IN.pts(), L.ptr(IN.n_pts()))),
    ("stage/frames_above_max_batch", "rgbl", CAP, lambda lib, h: lib.rgbl_resident_stage(h, 3, B + 1, _ptrs(IN.img + [IN.img[0]]), W, H, W, _ptrs(IN.clouds + [IN.clouds[0]]), L.ptr(np.append(IN.npts, 1).astype(np.int32)))),
    ("stage/cloud_above_max_points", "rgbl", CAP, lambda lib, h: lib.rgbl_resident_stage(h, 3, N, IN.g(), W, H, W, IN.pts(), L.ptr(IN.n_pts(f=1, value=NPTS + 1)))),
    ("stage/null_cloud", "rgbl", CAP, lambda lib, h: lib.rgbl_resident_stage(h, 3, N, IN.g(), W, H, W, IN.pts(null=0), L.ptr(IN.n_pts()))),
    # ---- RGB-L: sequence runner ----
    ("track_sequence/null_P", "rgbl", INV, lambda lib, h: _rgbl(lib, h, _seq_io(gray=IN.g(), pts=IN.pts(), n_pts=IN.n_pts()), P=None)),
    ("track_sequence/null_chain", "rgbl", INV, lambda lib, h: lib.rgbl_track_sequence(h, L.ptr(IN.P), C.byref(IN.prm), None, C.byref(_seq_io(gray=IN.g(), pts=IN.pts(), n_pts=IN.n_pts())))),
    ("track_sequence/null_clouds", "rgbl", INV, lambda lib, h: _rgbl(lib, h, _seq_io(gray=IN.g(), n_pts=IN.n_pts()))),
    ("track_sequence/frames_above_max_batch", "rgbl", INV, lambda lib, h: _rgbl(lib, h, _seq_io(T=B + 1, gray=_ptrs(IN.img + [IN.img[0]]), pts=_ptrs(IN.clouds + [IN.clouds[0]]), n_pts=np.append(IN.npts, 1).astype(np.int32)))),
    ("track_sequence/wrong_width", "rgbl", INV, lambda lib, h: _rgbl(lib, h, _seq_io(gray=IN.g(), pts=IN.pts(), n_pts=IN.n_pts(), width=W - 1, stride=W))),
    ("track_sequence/empty_image", "rgbl", EMPTY, lambda lib, h: _rgbl(lib, h, _seq_io(gray=IN.g(null=1), pts=IN.pts(), n_pts=IN.n_pts()))),
    ("track_sequence/cloud_above_max_points", "rgbl", CAP, lambda lib, h: _rgbl(lib, h, _seq_io(gray=IN.g(), pts=IN.pts(), n_pts=IN.n_pts(f=1, value=NPTS + 1)))),
    ("track_sequence/bad_frame_outputs", "rgbl", INV, lambda lib, h: _rgbl(lib, h, _seq_io_with_frames(_seq_io(gray=IN.g(), pts=IN.pts(), n_pts=IN.n_pts()), cap=7))),
    ("track_sequence/no_slots", "rgbl", INV, lambda lib, h: _rgbl(lib, h, _seq_io(n_slots=0))),
    ("track_sequence/nine_slots", "rgbl", INV, lambda lib, h: _rgbl(lib, h, _seq_io(n_slots=9))),
    ("track_sequence/empty_slot", "rgbl", INV, lambda lib, h: _rgbl(lib, h, _seq_io(n_slots=8, first_slot=SLOT_EMPTY))),
    ("track_sequence/rgbd_slot", "rgbl", INV, lambda lib, h: _rgbl(lib, h, _seq_io(n_slots=3, first_slot=SLOT_RGBD))),
    ("track_sequence/stereo_slot", "rgbl", INV, lambda lib, h: _rgbl(lib, h, _seq_io(n_slots=3, first_slot=SLOT_STEREO))),
    ("track_sequence/slot_of_other_size", "rgbl", INV, lambda lib, h: _rgbl(lib, h, _seq_io(T=1, n_slots=3, first_slot=SLOT_RGBL))),
    ("track_sequence/bad_depth_method_after_restage", "rgbl", UNSUP, lambda lib, h: _rgbl(lib, h, _seq_io(n_slots=3, first_slot=SLOT_RGBL), prm=_prm(method=9))),
    # ---- RGB-D: upload, PNG upload, decode ----
    ("upload_rgbd/null_gray", "rgbd", INV, lambda lib, h: lib.rgbl_resident_upload_rgbd(h, N, None, W, H, W, IN.d(), W)),
    ("upload_rgbd/null_depth", "rgbd", INV, lambda lib, h: lib.rgbl_resident_upload_rgbd(h, N, IN.g(), W, H, W, None, W)),
    ("upload_rgbd/empty_image", "rgbd", EMPTY, lambda lib, h: lib.rgbl_resident_upload_rgbd(h, N, IN.g(null=1), W, H, W, IN.d(), W)),
    ("upload_rgbd/empty_depth_image", "rgbd", EMPTY, lambda lib, h: lib.rgbl_resident_upload_rgbd(h, N, IN.g(), W, H, W, IN.d(null=0), W)),
    ("upload_rgbd/depth_stride_below_width", "rgbd", INV, lambda lib, h: lib.rgbl_resident_upload_rgbd(h, N, IN.g(), W, H, W, IN.d(), W - 1)),
    ("upload_rgbd/empty_image_and_depth_stride", "rgbd", EMPTY, lambda lib, h: lib.rgbl_resident_upload_rgbd(h, N, IN.g(null=0), W, H, W, IN.d(), W - 1)),
    ("upload_rgbd/stride_below_width", "rgbd", INV, lambda lib, h: lib.rgbl_resident_upload_rgbd(h, N, IN.g(), W, H, W - 1, IN.d(), W)),
    ("upload_rgbd/frames_above_max_batch", "rgbd", CAP, lambda lib, h: lib.rgbl_resident_upload_rgbd(h, B + 1, _ptrs(IN.img + [IN.img[0]]), W, H, W, _ptrs(IN.dep + [IN.dep[0]]), W)),
    ("upload_rgbd_png/null_depth_png", "rgbd", INV, lambda lib, h: lib.rgbl_resident_upload_rgbd_png(h, N, *_png_args(), 1, None, None)),
    ("upload_rgbd_png/empty_depth_stream", "rgbd", EMPTY, lambda lib, h: lib.rgbl_resident_upload_rgbd_png(h, N, *_png_args(), 1, *_png_args("dpng", empty=1))),
    ("upload_rgbd_png/wrong_depth_size", "rgbd", INV, lambda lib, h: lib.rgbl_resident_upload_rgbd_png(h, N, *_png_args(), 1, *_png_args("dpng", small=1))),
    ("upload_rgbd_png/8_bit_depth", "rgbd", UNSUP, lambda lib, h: lib.rgbl_resident_upload_rgbd_png(h, N, *_png_args(), 1, *_png_args())),
    ("upload_rgbd_png/frames_above_max_batch", "rgbd", CAP, lambda lib, h: lib.rgbl_resident_upload_rgbd_png(h, B + 1, *_png_args(n=B), 1, *_png_args("dpng", n=B))),
    ("decode_png_depth16/null_output", "rgbd", INV, lambda lib, h: lib.rgbl_decode_png_depth16(h, N, *_png_args("dpng"), _ptrs([None, np.empty((H, W), np.uint16)]), W)),
    # ---- RGB-D: process ----
    ("process_rgbd/nothing_of_this_kind", "rgbd", INV, _after("rgbl", lambda lib, h: lib.rgbl_resident_process_rgbd(h, DEPTH_SCALE, BF, None))),
    ("process_rgbd/after_stereo_upload", "rgbd", INV, _after("stereo", lambda lib, h: lib.rgbl_resident_process_rgbd(h, DEPTH_SCALE, BF, None))),
    ("process_rgbd/depth_scale_inf", "rgbd", INV, _after("rgbd", lambda lib, h: lib.rgbl_resident_process_rgbd(h, float("inf"), BF, None))),
    ("process_rgbd/bf_zero", "rgbd", INV, _after("rgbd", lambda lib, h: lib.rgbl_resident_process_rgbd(h, DEPTH_SCALE, 0.0, None))),
    ("process_rgbd/bf_nan", "rgbd", INV, _after("rgbd", lambda lib, h: lib.rgbl_resident_process_rgbd(h, DEPTH_SCALE, float("nan"), None))),
    # ---- RGB-D: stage ----
    ("stage_rgbd/slot_above_range", "rgbd", INV, lambda lib, h: lib.rgbl_resident_stage_rgbd(h, 8, N, IN.g(), W, H, W, IN.d(), W)),
    ("stage_rgbd/null_depth", "rgbd", INV, lambda lib, h: lib.rgbl_resident_stage_rgbd(h, 3, N, IN.g(), W, H, W, None, W)),
    ("stage_rgbd/empty_depth_image", "rgbd", EMPTY, lambda lib, h: lib.rgbl_resident_stage_rgbd(h, 3, N, IN.g(), W, H, W, IN.d(null=1), W)),
    ("stage_rgbd/empty_image", "rgbd", EMPTY, lambda lib, h: lib.rgbl_resident_stage_rgbd(h, 3, N, IN.g(null=0), W, H, W, IN.d(), W)),
    ("stage_rgbd/depth_stride_below_width", "rgbd", INV, lambda lib, h: lib.rgbl_resident_stage_rgbd(h, 3, N, IN.g(), W, H, W, IN.d(), W - 1)),
    ("stage_rgbd/depth_stride_and_empty_image", "rgbd", INV, lambda lib, h: lib.rgbl_resident_stage_rgbd(h, 3, N, IN.g(null=0), W, H, W, IN.d(), W - 1)),
    ("stage_rgbd/frames_above_max_batch", "rgbd", CAP, lambda lib, h: lib.rgbl_resident_stage_rgbd(h, 3, B + 1, _ptrs(IN.img + [IN.img[0]]), W, H, W, _ptrs(IN.dep + [IN.dep[0]]), W)),
    # ---- RGB-D: sequence runner ----
    ("track_sequence_rgbd/depth_scale_nan", "rgbd", INV, lambda lib, h: _rgbd(lib, h, _seq_io(gray=IN.g()), IN.d(), depth_scale=float("nan"))),
    ("track_sequence_rgbd/bf_negative", "rgbd", INV, lambda lib, h: _rgbd(lib, h, _seq_io(gray=IN.g()), IN.d(), bf=-1.0)),
    ("track_sequence_rgbd/point_clouds", "rgbd", INV, lambda lib, h: _rgbd(lib, h, _seq_io(gray=IN.g(), pts=IN.pts(), n_pts=IN.n_pts()), IN.d())),
    ("track_sequence_rgbd/null_depth", "rgbd", INV, lambda lib, h: _rgbd(lib, h, _seq_io(gray=IN.g()), None)),
    ("track_sequence_rgbd/depth_stride_below_width", "rgbd", INV, lambda lib, h: _rgbd(lib, h, _seq_io(gray=IN.g()), IN.d(), depth_stride=W - 1)),
    ("track_sequence_rgbd/empty_image", "rgbd", EMPTY, lambda lib, h: _rgbd(lib, h, _seq_io(gray=IN.g(null=1)), IN.d())),
    ("track_sequence_rgbd/empty_depth_image", "rgbd", EMPTY, lambda lib, h: _rgbd(lib, h, _seq_io(gray=IN.g()), IN.d(null=1))),
    ("track_sequence_rgbd/frames_above_max_batch", "rgbd", INV, lambda lib, h: _rgbd(lib, h, _seq_io(T=B + 1, gray=_ptrs(IN.img + [IN.img[0]])), _ptrs(IN.dep + [IN.dep[0]]))),
    ("track_sequence_rgbd/empty_slot", "rgbd", INV, lambda lib, h: _rgbd(lib, h, _seq_io(n_slots=8, first_slot=SLOT_EMPTY))),
    ("track_sequence_rgbd/rgbl_slot", "rgbd", INV, lambda lib, h: _rgbd(lib, h, _seq_io(n_slots=3, first_slot=SLOT_RGBL))),
    ("track_sequence_rgbd/stereo_slot", "rgbd", INV, lambda lib, h: _rgbd(lib, h, _seq_io(n_slots=3, first_slot=SLOT_STEREO))),
    ("track_sequence_rgbd/slot_of_other_size", "rgbd", INV, lambda lib, h: _rgbd(lib, h, _seq_io(T=1, n_slots=3, first_slot=SLOT_RGBD))),
    # ---- stereo: upload, PNG upload ----
    ("upload_stereo/null_right", "stereo", INV, lambda lib, h: lib.rgbl_resident_upload_stereo(h, N, IN.g(), None, W, H, W)),
    ("upload_stereo/empty_left", "stereo", EMPTY, lambda lib, h: lib.rgbl_resident_upload_stereo(h, N, IN.g(null=1), IN.r(), W, H, W)),
    ("upload_stereo/empty_right", "stereo", EMPTY, lambda lib, h: lib.rgbl_resident_upload_stereo(h, N, IN.g(), IN.r(null=0), W, H, W)),
    ("upload_stereo/wrong_width", "stereo", INV, lambda lib, h: lib.rgbl_resident_upload_stereo(h, N, IN.g(), IN.r(), W - 4, H, W)),
    ("upload_stereo/pairs_above_half_max_batch", "stereo", INV, lambda lib, h: lib.rgbl_resident_upload_stereo(h, 3, IN.g(3), IN.r(3), W, H, W)),
    ("upload_stereo/pairs_above_max_batch", "stereo", CAP, lambda lib, h: lib.rgbl_resident_upload_stereo(h, B + 1, _ptrs(IN.img + [IN.img[0]]), _ptrs(IN.right + [IN.right[0]]), W, H, W)),
    ("upload_stereo/distorted_camera", "stereo", UNSUP, _distorted(lambda lib, h: lib.rgbl_resident_upload_stereo(h, N, IN.g(), IN.r(), W, H, W))),
    ("upload_stereo/distorted_camera_and_empty_image", "stereo", UNSUP, _distorted(lambda lib, h: lib.rgbl_resident_upload_stereo(h, N, IN.g(null=0), IN.r(), W, H, W))),
    ("upload_stereo_png/null_right", "stereo", INV, lambda lib, h: lib.rgbl_resident_upload_stereo_png(h, N, *_png_args(), None, None, 1)),
    ("upload_stereo_png/empty_right_stream", "stereo", EMPTY, lambda lib, h: lib.rgbl_resident_upload_stereo_png(h, N, *_png_args(), *_png_args("rpng", empty=1), 1)),
    ("upload_stereo_png/right_of_other_size", "stereo", INV, lambda lib, h: lib.rgbl_resident_upload_stereo_png(h, N, *_png_args(), *_png_args("rpng", small=1), 1)),
    ("upload_stereo_png/pairs_above_half_max_batch", "stereo", INV, lambda lib, h: lib.rgbl_resident_upload_stereo_png(h, 3, *_png_args(n=3), *_png_args("rpng", n=3), 1)),
    ("upload_stereo_png/distorted_camera", "stereo", UNSUP, _distorted(lambda lib, h: lib.rgbl_resident_upload_stereo_png(h, N, *_png_args(), *_png_args("rpng"), 1))),
    # ---- stereo: process ----
    ("process_stereo/after_rgbl_upload", "stereo", INV, _after("rgbl", lambda lib, h: lib.rgbl_resident_process_stereo(h, MB, MBF, None))),
    ("process_stereo/after_rgbd_upload", "stereo", INV, _after("rgbd", lambda lib, h: lib.rgbl_resident_process_stereo(h, MB, MBF, None))),
    ("process_stereo/mb_zero", "stereo", INV, _after("stereo", lambda lib, h: lib.rgbl_resident_process_stereo(h, 0.0, MBF, None))),
    ("process_stereo/mbf_inf", "stereo", INV, _after("stereo", lambda lib, h: lib.rgbl_resident_process_stereo(h, MB, float("inf"), None))),
    ("process_stereo/distorted_camera", "stereo", UNSUP, _after("stereo", _distorted(lambda lib, h: lib.rgbl_resident_process_stereo(h, MB, MBF, None)))),
    ("process_stereo/distorted_camera_and_mb_nan", "stereo", INV, _after("stereo", _distorted(lambda lib, h: lib.rgbl_resident_process_stereo(h, float("nan"), MBF, None)))),
    # ---- stereo: stage ----
    ("stage_stereo/slot_below_range", "stereo", INV, lambda lib, h: lib.rgbl_resident_stage_stereo(h, -1, N, IN.g(), IN.r(), W, H, W)),
    ("stage_stereo/null_left", "stereo", INV, lambda lib, h: lib.rgbl_resident_stage_stereo(h, 3, N, None, IN.r(), W, H, W)),
    ("stage_stereo/empty_right", "stereo", EMPTY, lambda lib, h: lib.rgbl_resident_stage_stereo(h, 3, N, IN.g(), IN.r(null=1), W, H, W)),
    ("stage_stereo/pairs_above_half_max_batch", "stereo", INV, lambda lib, h: lib.rgbl_resident_stage_stereo(h, 3, 3, IN.g(3), IN.r(3), W, H, W)),
    ("stage_stereo/stride_below_width", "stereo", INV, lambda lib, h: lib.rgbl_resident_stage_stereo(h, 3, N, IN.g(), IN.r(), W, H, W - 1)),
    ("stage_stereo/distorted_camera", "stereo", UNSUP, _distorted(lambda lib, h: lib.rgbl_resident_stage_stereo(h, 3, N, IN.g(), IN.r(), W, H, W))),
    # ---- stereo: sequence runner ----
    ("track_sequence_stereo/mb_negative", "stereo", INV, lambda lib, h: _stereo(lib, h, _seq_io(gray=IN.g()), IN.r(), mb=-1.0)),
    ("track_sequence_stereo/mbf_nan", "stereo", INV, lambda lib, h: _stereo(lib, h, _seq_io(gray=IN.g()), IN.r(), mbf=float("nan"))),
    ("track_sequence_stereo/point_clouds", "stereo", INV, lambda lib, h: _stereo(lib, h, _seq_io(gray=IN.g(), pts=IN.pts()), IN.r())),
    ("track_sequence_stereo/null_right", "stereo", INV, lambda lib, h: _stereo(lib, h, _seq_io(gray=IN.g()), None)),
    ("track_sequence_stereo/empty_right", "stereo", EMPTY, lambda lib, h: _stereo(lib, h, _seq_io(gray=IN.g()), IN.r(null=1))),
    ("track_sequence_stereo/pairs_above_half_max_batch", "stereo", INV, lambda lib, h: _stereo(lib, h, _seq_io(T=3, gray=IN.g(3)), IN.r(3))),
    ("track_sequence_stereo/distorted_camera", "stereo", UNSUP, _distorted(lambda lib, h: _stereo(lib, h, _seq_io(gray=IN.g()), IN.r()))),
    ("track_sequence_stereo/empty_slot", "stereo", INV, lambda lib, h: _stereo(lib, h, _seq_io(n_slots=8, first_slot=SLOT_EMPTY))),
    ("track_sequence_stereo/rgbl_slot", "stereo", INV, lambda lib, h: _stereo(lib, h, _seq_io(n_slots=3, first_slot=SLOT_RGBL))),
    ("track_sequence_stereo/rgbd_slot", "stereo", INV, lambda lib, h: _stereo(lib, h, _seq_io(n_slots=3, first_slot=SLOT_RGBD))),
    ("track_sequence_stereo/slot_of_other_size", "stereo", INV, lambda lib, h: _stereo(lib, h, _seq_io(T=1, n_slots=3, first_slot=SLOT_STEREO))),
    ("track_sequence_stereo/distorted_camera_and_rgbl_slot", "stereo", UNSUP, _distorted(lambda lib, h: _stereo(lib, h, _seq_io(n_slots=3, first_slot=SLOT_RGBL)))),
]


def _seq_io_with_frames(io, cap):
    """io with frame outputs of capacity `cap`."""
    n = io.frames_per_batch * io.n_batches
    arrs = [np.empty((n, cap), L.KP_DTYPE), np.empty((n, cap, 32), np.uint8), np.empty((n, cap), np.float32), np.empty((n, cap), np.float32), np.zeros(n, np.int32)]
    io._keep += arrs
    io.kps, io.desc, io.depth, io.uright = (a.ctypes.data for a in arrs[:4])
    io.cap, io.n_kp = cap, arrs[4].ctypes.data
    return io


@pytest.fixture(scope="module")
def shared(lib):
    """A context with slots 0..2 staged, and the outputs of a fresh context for each kind."""
    ref = {}
    for kind in ("rgbl", "rgbd", "stereo"):
        h = _new_ctx(lib)
        ref[kind] = _build(lib, h, kind)
        lib.rgbl_destroy(h)
    h = _new_ctx(lib)
    assert lib.rgbl_resident_stage(h, SLOT_RGBL, N, IN.g(), W, H, W, IN.pts(), L.ptr(IN.n_pts())) == 0
    assert lib.rgbl_resident_stage_rgbd(h, SLOT_RGBD, N, IN.g(), W, H, W, IN.d(), W) == 0
    assert lib.rgbl_resident_stage_stereo(h, SLOT_STEREO, N, IN.g(), IN.r(), W, H, W) == 0
    yield h, ref
    lib.rgbl_destroy(h)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_refused_call_keeps_the_context_usable(lib, shared, case):
    _, kind, status, call = case
    h, ref = shared
    assert call(lib, h) == status, lib.rgbl_last_error(h)
    assert _build(lib, h, kind) == ref[kind]


def test_nothing_uploaded_and_no_point_clouds(lib, shared):
    """A fresh context refuses the process calls (nothing uploaded); one created with max_points == 0 refuses every RGB-L input and
    still builds RGB-D and stereo frames."""
    _, ref = shared
    h = _new_ctx(lib)
    try:
        assert lib.rgbl_resident_process(h, L.ptr(IN.P), C.byref(IN.prm), None) == INV
        assert lib.rgbl_resident_process_rgbd(h, DEPTH_SCALE, BF, None) == INV
        assert lib.rgbl_resident_process_stereo(h, MB, MBF, None) == INV
        assert _build(lib, h, "stereo") == ref["stereo"]
    finally:
        lib.rgbl_destroy(h)
    h = _new_ctx(lib, max_points=0)
    try:
        assert _frame_rgbl(lib, h, n_pts=np.zeros(N, np.int32)) == INV
        assert lib.rgbl_resident_upload(h, N, IN.g(), W, H, W, IN.pts(), L.ptr(np.zeros(N, np.int32))) == INV
        assert lib.rgbl_resident_upload_kitti(h, N, IN.g(), W, H, W, IN.kitti(), L.ptr(np.zeros(N, np.int32))) == INV
        assert lib.rgbl_resident_upload_kitti_png(h, N, *_png_args(), 1, IN.kitti(), L.ptr(np.zeros(N, np.int32))) == INV
        assert lib.rgbl_resident_stage(h, 0, N, IN.g(), W, H, W, IN.pts(), L.ptr(np.zeros(N, np.int32))) == INV
        assert _rgbl(lib, h, _seq_io(gray=IN.g(), pts=IN.pts(), n_pts=np.zeros(N, np.int32))) == INV
        assert _rgbl(lib, h, _seq_io(n_slots=1)) == INV
        assert _build(lib, h, "rgbd") == ref["rgbd"]
        assert _build(lib, h, "stereo") == ref["stereo"]
    finally:
        lib.rgbl_destroy(h)


def test_rectified_stereo_refusals(lib, shared):
    """With rectification on (identity maps, so the rectified pairs are the pairs themselves): a colour PNG is refused before anything
    is copied, the refusals of the other stereo calls are unchanged, and the context still builds the frames of a fresh context."""
    h, ref = shared
    xs, ys = np.meshgrid(np.arange(W, dtype=np.float32), np.arange(H, dtype=np.float32))
    assert lib.rgbl_set_stereo_rectification(h, L.ptr(xs), L.ptr(ys), L.ptr(xs), L.ptr(ys), W) == 0
    try:
        colour = [np.frombuffer(S.encode_png(S.colorize(i)), np.uint8) for i in IN.img[:N]]
        assert lib.rgbl_resident_upload_stereo_png(h, N, _ptrs(colour), _sizes(colour), *_png_args("rpng"), 1) == UNSUP
        assert lib.rgbl_resident_process_stereo(h, MB, MBF, None) == INV         # setting the maps discarded the uploaded pairs
        assert lib.rgbl_resident_upload_stereo(h, N, IN.g(), IN.r(null=1), W, H, W) == EMPTY
        assert lib.rgbl_resident_upload_stereo(h, 3, IN.g(3), IN.r(3), W, H, W) == INV
        assert _stereo(lib, h, _seq_io(n_slots=3, first_slot=SLOT_RGBD)) == INV
        assert _stereo(lib, h, _seq_io(T=1, n_slots=3, first_slot=SLOT_STEREO)) == INV
        assert _build(lib, h, "stereo") == ref["stereo"]
        p, s, keep = IN.pngs("png"); rp, rs, rkeep = IN.pngs("rpng")
        cnt = np.zeros(N, np.int32)
        assert lib.rgbl_resident_upload_stereo_png(h, N, p, s, rp, rs, 1) == 0
        assert lib.rgbl_resident_process_stereo(h, MB, MBF, L.ptr(cnt)) == 0
        assert _download(lib, h, N) == ref["stereo"]
    finally:
        assert lib.rgbl_set_stereo_rectification(h, None, None, None, None, 0) == 0
    assert _build(lib, h, "stereo") == ref["stereo"]

"""Sequence lanes (rgbl_set_sequences) against the whole library compiled over the CUDA-on-CPU shim (tests/cuda_emu): a context that tracks
S sequences in lockstep must give every lane, bit for bit, what a one-lane context gives for that lane's frames alone; lanes never
read each other's state; and every refusal of the setting and of the lane geometry returns RGBL_E_INVALID."""
import ctypes as C

import numpy as np
import pytest

from cuda_emu import build
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S

W, H, NPTS = 160, 120, 400
FX, FY, CX, CY, BF = 100.0, 100.0, 80.0, 60.0, 40.0
DEPTH_SCALE = 0.001
INV = L.RGBL_E_INVALID
M = 2                                  # frames per lane per batch
NB = 3                                 # batches: each after the first continues the sequences


@pytest.fixture(scope="module")
def lib():
    so = C.CDLL(str(build.build_full()))
    for name, (res, args) in L.SYMBOLS.items():
        fn = getattr(so, name)
        fn.restype, fn.argtypes = res, args
    return so


def _ctx(lib, max_batch):
    cfg = L.Config(0, W, H, max_batch, NPTS, 0, L.OrbParams(200, 1.2, 4, 20, 7))
    h = C.c_void_p()
    assert lib.rgbl_create(C.byref(cfg), C.byref(h)) == 0
    assert lib.rgbl_set_host_quadtree(h, 1) == 0
    return h


def _depth_params():
    p = L.DepthParams()
    p.method, p.min_dist, p.max_dist, p.bf, p.inv_dilation_scale = L.DEPTH_INVERSE_DILATION, 5.0, 200.0, BF, 1.0
    p.ku = p.kv = 5
    flat = np.zeros(81, np.uint8); flat[:25] = S.structuring_element("diamond", 5).reshape(-1)
    C.memmove(p.mask, flat.ctypes.data, 81)
    p.avg_kernel, p.nn_search_radius = 5, 7.0
    return p


PRM = _depth_params()
P12 = np.array([[FX, 0, CX, 0], [0, FY, CY, 0], [0, 0, 1, 0]], np.float32).reshape(12)


class Lane:
    """One sequence of NB * M frames: an image drifting one pixel per frame, a fixed cloud (no depth: an empty cloud), depth images."""

    def __init__(self, seed, depth=True):
        rng = np.random.default_rng(seed)
        base = S.make_image(seed, W + 16, H, 40)
        self.img = [np.ascontiguousarray(base[:, f:f + W]) for f in range(NB * M)]
        self.right = [np.ascontiguousarray(np.roll(i, -3, axis=1)) for i in self.img]
        n = 300 if depth else 0
        z = rng.uniform(6.0, 40.0, n)
        x = (rng.uniform(0, W, n) - CX) * z / FX; y = (rng.uniform(0, H, n) - CY) * z / FY
        cloud = np.ascontiguousarray(np.stack([x, y, z, np.ones(n)]).astype(np.float32).reshape(4, n))
        self.clouds = [cloud] * (NB * M)
        d = rng.integers(1000, 20000, (H, W)).astype(np.uint16) if depth else np.zeros((H, W), np.uint16)
        self.dep = [d] * (NB * M)


def _interleave(lanes, attr):
    """the frames of all lanes in batch order: batch b, lane s, frame k"""
    S_ = len(lanes)
    return [getattr(lanes[s], attr)[b * M + k] for b in range(NB) for s in range(S_) for k in range(M)]


_KEEP = []


def _ptrs(arrays):
    _KEEP.append(arrays)
    return (C.c_void_p * len(arrays))(*[a.ctypes.data for a in arrays])


def _run(lib, kind, lanes, K, pose0):
    """rgbl_track_sequence* of the lanes (host mode, NB continuing batches of S * M frames) on a fresh context -> poses, counters"""
    S_ = len(lanes)
    T = S_ * M
    h = _ctx(lib, 2 * T if kind == "stereo" else T)          # a stereo batch of T pairs takes 2 T frame slots
    try:
        p0 = np.ascontiguousarray(pose0, np.float32)
        assert lib.rgbl_set_sequences(h, S_, L.ptr(p0)) == 0
        imgs = _interleave(lanes, "img")
        io = F.SequenceIO()
        io.n_batches, io.frames_per_batch, io.width, io.height, io.stride = NB, T, W, H, W
        gray = _ptrs(imgs)
        io.gray = C.cast(gray, C.c_void_p)
        out = [np.zeros((NB * T, 7), np.float32)] + [np.zeros(NB * T, np.int32) for _ in range(3)]
        _KEEP.append(out)
        io.poses, io.n_matches, io.n_inliers, io.n_local_matches = (a.ctypes.data for a in out)
        chain = F.make_chain_params([0, 0, 0, 1, 0, 0, 0], FX, FY, CX, CY, BF, local_map_frames=K)
        if kind == "rgbl":
            clouds = _interleave(lanes, "clouds")
            io.pts4xn = C.cast(_ptrs(clouds), C.c_void_p)
            npts = np.array([c.shape[1] for c in clouds], np.int32); _KEEP.append(npts)
            io.n_pts = npts.ctypes.data
            rc = lib.rgbl_track_sequence(h, L.ptr(P12), C.byref(PRM), C.byref(chain), C.byref(io))
        elif kind == "rgbd":
            rc = lib.rgbl_track_sequence_rgbd(h, DEPTH_SCALE, BF, C.byref(chain), C.byref(io), _ptrs(_interleave(lanes, "dep")), W)
        else:
            rc = lib.rgbl_track_sequence_stereo(h, 0.4, BF, C.byref(chain), C.byref(io), _ptrs(_interleave(lanes, "right")))
        assert rc == 0, rc
        return out
    finally:
        lib.rgbl_destroy(h)


def _lane_of(out, S_, s):
    """lane s's frames of a run with S_ lanes, in sequence order"""
    idx = [b * S_ * M + s * M + k for b in range(NB) for k in range(M)]
    return [a[idx] for a in out]


def _pose0(S_):
    p = np.zeros((S_, 7), np.float32)
    p[:, 3] = 1.0
    p[:, 4] = 0.01 * np.arange(S_); p[:, 6] = -0.02 * np.arange(S_)
    return p


def _check_lanes(lib, kind, lanes, K):
    S_ = len(lanes)
    p0 = _pose0(S_)
    multi = _run(lib, kind, lanes, K, p0)
    for s in range(S_):
        single = _run(lib, kind, [lanes[s]], K, p0[s:s + 1])
        got = _lane_of(multi, S_, s)
        for name, a, b in zip(("poses", "n_matches", "n_inliers", "n_local_matches"), got, single):
            assert a.tobytes() == b.tobytes(), f"lane {s}: {name} differs from the one-lane run"
    return multi


@pytest.mark.parametrize("S_,K", [(2, 0), (2, 2), (3, 0), (3, 2)])
def test_lanes_equal_single_sequence_rgbl(lib, S_, K):
    out = _check_lanes(lib, "rgbl", [Lane(40 + 3 * s) for s in range(S_)], K)
    assert out[1].max() > 0                 # the lanes did match something


@pytest.mark.parametrize("kind", ["rgbd", "stereo"])
def test_lanes_equal_single_sequence_rgbd_stereo(lib, kind):
    _check_lanes(lib, kind, [Lane(61), Lane(67)], 2)


def test_identical_lanes_identical_outputs(lib):
    out = _run(lib, "rgbl", [Lane(50), Lane(50)], 2, np.tile(_pose0(1), (2, 1)))
    a, b = _lane_of(out, 2, 0), _lane_of(out, 2, 1)
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()


def test_empty_lane_leaves_other_lanes_unchanged(lib):
    p0 = _pose0(2)
    with_depth = _run(lib, "rgbl", [Lane(52), Lane(53)], 2, p0)
    empty = _run(lib, "rgbl", [Lane(52), Lane(53, depth=False)], 2, p0)
    for x, y in zip(_lane_of(with_depth, 2, 0), _lane_of(empty, 2, 0)):
        assert x.tobytes() == y.tobytes()


def _manual(lib, lanes, K, pose0):
    """rgbl_resident_track_begin2 / _end2 over NB batches (the chains of consecutive batches queued two deep) -> the five per-frame outputs"""
    S_ = len(lanes)
    T = S_ * M
    h = _ctx(lib, T)
    try:
        p0 = np.ascontiguousarray(pose0, np.float32)
        assert lib.rgbl_set_sequences(h, S_, L.ptr(p0)) == 0
        imgs, clouds = _interleave(lanes, "img"), _interleave(lanes, "clouds")
        out = [np.zeros((NB * T, 7), np.float32)] + [np.zeros(NB * T, np.int32) for _ in range(4)]
        _KEEP.append(out)
        pending = []
        for b in range(NB):
            fr = slice(b * T, (b + 1) * T)
            npts = np.array([c.shape[1] for c in clouds[fr]], np.int32); _KEEP.append(npts)
            assert lib.rgbl_resident_upload(h, T, _ptrs(imgs[fr]), W, H, W, _ptrs(clouds[fr]), npts.ctypes.data) == 0
            assert lib.rgbl_resident_process(h, L.ptr(P12), C.byref(PRM), None) == 0
            chain = F.make_chain_params([0, 0, 0, 1, 0, 0, 0], FX, FY, CX, CY, BF, continue_sequence=b > 0, local_map_frames=K)
            assert lib.rgbl_resident_track_begin2(h, C.byref(chain)) == 0
            pending.append(b)
            if len(pending) == 2 or b == NB - 1:
                while pending:
                    o = pending.pop(0) * T
                    ptrs = [out[0][o:].ctypes.data] + [a[o:].ctypes.data for a in out[1:]]
                    assert lib.rgbl_resident_track_end2(h, *ptrs) == 0
        return out
    finally:
        lib.rgbl_destroy(h)


def test_manual_chain_lanes_equal_single_sequence(lib):
    """the manual chain API with two chains queued; n_inliers_first (not a runner output) is compared too"""
    lanes, p0 = [Lane(44), Lane(45)], _pose0(2)
    multi = _manual(lib, lanes, 2, p0)
    for s in range(2):
        single = _manual(lib, [lanes[s]], 2, p0[s:s + 1])
        for name, a, b in zip(("poses", "n_matches", "n_inliers", "n_local_matches", "n_inliers_first"), _lane_of(multi, 2, s), single):
            assert a.tobytes() == b.tobytes(), f"lane {s}: {name} differs from the one-lane run"


# Each refusal: call(lib, h, bad) returns the status of the faulty call (bad=True) or of the same call made valid (bad=False, the positive
# control on a fresh context), and the error text the refusal must give.
def _refusals():
    def n_seq(n_bad, n_good):
        return lambda lib, h, bad: lib.rgbl_set_sequences(h, n_bad if bad else n_good, None)

    def pose0(lib, h, bad):
        p = _pose0(2)
        if bad:
            p[1, 5] = np.nan
        return lib.rgbl_set_sequences(h, 2, L.ptr(p))

    def setting_kept(lib, h, bad):
        assert lib.rgbl_set_sequences(h, 2, None) == 0
        assert lib.rgbl_set_sequences(h, 0, None) == INV
        # the refused call left 2 lanes: a 3-frame batch is not a multiple of them, a 4-frame one is
        return _chain(lib, h, 3 if bad else 4, cont=False)

    def batch_not_multiple(lib, h, bad):
        assert lib.rgbl_set_sequences(h, 2 if bad else 1, None) == 0
        return _chain(lib, h, 3, cont=False)

    def runner_not_multiple(lib, h, bad):
        assert lib.rgbl_set_sequences(h, 2 if bad else 1, None) == 0
        lane = Lane(70)
        io = F.SequenceIO()
        io.n_batches, io.frames_per_batch, io.width, io.height, io.stride = 1, 3, W, H, W
        io.gray = C.cast(_ptrs(lane.img[:3]), C.c_void_p)
        io.pts4xn = C.cast(_ptrs(lane.clouds[:3]), C.c_void_p)
        npts = np.full(3, lane.clouds[0].shape[1], np.int32); _KEEP.append(npts)
        io.n_pts = npts.ctypes.data
        out = [np.zeros((3, 7), np.float32), np.zeros(3, np.int32), np.zeros(3, np.int32)]; _KEEP.append(out)
        io.poses, io.n_matches, io.n_inliers = (a.ctypes.data for a in out)
        chain = F.make_chain_params([0, 0, 0, 1, 0, 0, 0], FX, FY, CX, CY, BF)
        return lib.rgbl_track_sequence(h, L.ptr(P12), C.byref(PRM), C.byref(chain), C.byref(io))

    def continue_other_lane_count(lib, h, bad):
        assert lib.rgbl_set_sequences(h, 2, None) == 0
        assert _chain(lib, h, 4, cont=False) == 0
        assert lib.rgbl_set_sequences(h, 1 if bad else 2, None) == 0
        return _chain(lib, h, 4, cont=True)

    bound = "n_sequences must be 1..16"
    return [
        ("zero_sequences", n_seq(0, 1), bound),
        ("above_bound", n_seq(17, 16), bound),                        # RGBL_MAX_SEQUENCES = 16
        ("non_finite_pose0", pose0, "non-finite"),
        ("refused_setting_keeps_previous", setting_kept, "not a multiple of the sequence count"),
        ("batch_not_multiple", batch_not_multiple, "not a multiple of the sequence count"),
        ("runner_frames_per_batch_not_multiple", runner_not_multiple, "frames_per_batch is not a multiple of the sequence count"),
        ("continue_with_other_lane_count", continue_other_lane_count, "sequence count differs from the previous chain"),
    ]


def _chain(lib, h, n, cont):
    """process n frames of one lane's images, then one chain through _begin2 / _end2"""
    lane = Lane(71)
    npts = np.full(n, lane.clouds[0].shape[1], np.int32); _KEEP.append(npts)
    assert lib.rgbl_resident_upload(h, n, _ptrs(lane.img[:n]), W, H, W, _ptrs(lane.clouds[:n]), npts.ctypes.data) == 0
    assert lib.rgbl_resident_process(h, L.ptr(P12), C.byref(PRM), None) == 0
    chain = F.make_chain_params([0, 0, 0, 1, 0, 0, 0], FX, FY, CX, CY, BF, continue_sequence=cont, local_map_frames=2)
    rc = lib.rgbl_resident_track_begin2(h, C.byref(chain))
    if rc:
        return rc
    out = [np.zeros((n, 7), np.float32), np.zeros(n, np.int32), np.zeros(n, np.int32)]
    return lib.rgbl_resident_track_end2(h, *[a.ctypes.data for a in out], None, None)


@pytest.mark.parametrize("name,call,text", _refusals(), ids=[r[0] for r in _refusals()])
def test_refusals(lib, name, call, text):
    for bad in (True, False):
        h = _ctx(lib, 4)
        try:
            rc = call(lib, h, bad)
            if bad:
                msg = (lib.rgbl_last_error(h) or b"").decode()
                assert rc == INV and text in msg, (rc, msg)
            else:
                assert rc == 0, (rc, (lib.rgbl_last_error(h) or b"").decode())
        finally:
            lib.rgbl_destroy(h)

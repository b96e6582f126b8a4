"""The DEVICE code paths of the kernel variants that have not run on a GPU yet, executed on the CUDA-on-CPU shim
(tests/cuda_emu: one OS thread per CUDA thread, real barriers, warp collectives as rendezvous) and compared with the oracle.
The host twins (tests/test_host_abi.py) check the algorithms; this checks the device-only glue around them: shuffle scans,
shared-memory atomics, warp reductions, dynamic shared-memory carving and the launch geometry."""
import ctypes as C

import numpy as np
import pytest

import oracle
from cuda_emu import build
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import synthetic as S


@pytest.fixture(scope="module")
def emu():
    lib = C.CDLL(str(build.build_full()))
    vp, i = C.c_void_p, C.c_int
    lib.emu_fast_strips.argtypes = [vp, i, i, i, vp, i, i, i, vp, i]
    lib.emu_describe_staged.argtypes = [vp, vp, vp, i, i, i, i, vp, vp, vp]
    lib.emu_quadtree.argtypes = [vp, i, i, i, i, vp, i]
    lib.emu_tlm_check.argtypes = [C.c_uint]
    return lib


def test_strip_fast_kernel_device_path(emu):
    w, h = 420, 240
    img = S.make_image(77, w, h)
    ex = oracle.Extractor(800); ex(img)
    prm = L.OrbParams(800, 1.2, 8, 12, 7)
    for l, (mc, mw) in zip((0, 2, 5), ((8, 264), (3, 130), (8, 264))):
        lv = ex.level_image(l)
        out = np.empty((1 << 15, 3), np.int32)
        n = emu.emu_fast_strips(C.byref(prm), w, h, l, L.ptr(lv), lv.strides[0], mc, mw, L.ptr(out), len(out))
        ref = ex.level_candidates(l)
        assert n == len(ref) and (out[:n] == ref).all(), l


def test_strip_fast_kernel_device_path_kitti_size(emu):
    """Full-width strips (8 cells, 258 px) of the KITTI level-0 geometry, a threshold pair that makes most cells fall back to
    minTh, and a tall-cell geometry (one cell row of 69 + 6 rows)."""
    for (w, h), ths, l in (((1241, 376), (12, 7), 0), ((1241, 376), (60, 7), 1), ((640, 302), (12, 7), 6)):
        img = S.make_image(91, w, h)
        ex = oracle.Extractor(1000, ini_th=ths[0], min_th=ths[1]); ex(img)
        prm = L.OrbParams(1000, 1.2, 8, ths[0], ths[1])
        lv = ex.level_image(l)
        out = np.empty((1 << 16, 3), np.int32)
        n = emu.emu_fast_strips(C.byref(prm), w, h, l, L.ptr(lv), lv.strides[0], 8, 264, L.ptr(out), len(out))
        ref = ex.level_candidates(l)
        assert n == len(ref) and (out[:n] == ref).all(), (w, h, l)


def test_staged_describe_kernel_device_path(emu):
    w, h = 420, 240
    img = S.make_image(78, w, h)
    ex = oracle.Extractor(300)
    kps, desc, _ = ex(img)
    prm = L.OrbParams(300, 1.2, 8, 12, 7)
    base = 0
    for l in range(8):
        kl = ex.level_keypoints(l)
        n = len(kl)
        if l in (0, 3) and n:
            lv = ex.level_image(l); bl = oracle.gaussian_blur7(lv)
            xy = np.ascontiguousarray(np.stack([kl["x"], kl["y"]], 1).astype(np.int32))
            ang = np.empty(n, np.float32); d = np.empty((n, 32), np.uint8)
            assert emu.emu_describe_staged(C.byref(prm), L.ptr(lv), L.ptr(bl), lv.shape[1], lv.shape[0], lv.strides[0], n, L.ptr(xy), L.ptr(ang), L.ptr(d)) == 0
            assert (ang.view(np.uint32) == np.ascontiguousarray(kps["angle"][base:base + n]).view(np.uint32)).all()
            assert (d == desc[base:base + n]).all()
        base += n


def test_quadtree_kernel_with_block_sort_device_path(emu):
    img = S.make_image(79, 700, 260)
    ex = oracle.Extractor(1000); ex(img)
    for l in (0, 4, 5):
        cand = np.ascontiguousarray(ex.level_candidates(l), np.int32)
        hh, ww = ex.level_image(l).shape
        nd = int(ex.features_per_level[l])
        out = np.empty((nd + 64, 3), np.int32)
        m = emu.emu_quadtree(L.ptr(cand), len(cand), ww, hh, nd, L.ptr(out), len(out))
        ref = ex.level_keypoints(l)
        assert m == len(ref)
        assert (out[:m, 0] == ref["x"]).all() and (out[:m, 1] == ref["y"]).all() and (out[:m, 2] == ref["response"]).all()


def test_depth_dilate_kernels_device_path(emu):
    """depth_project + depth_resolve_dilate_v2 (empty-tile shortcut, shared-memory tap offsets, the 5x5 diamond compiled in) against
    the oracle's ProjectPointcloudToImage + Upsample_InverseDilation, bit for bit; the cloud covers only the lower part of the image
    so that whole tiles are empty."""
    W, H = 333, 150
    P = S.lidar_projection_matrix().astype(np.float32)
    pts = S.make_pointcloud(3, n_azimuth=500)
    emu.emu_depth_dilate.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float,
                                     C.c_float, C.c_void_p, C.c_void_p]
    # shift the projection so that the returns land inside this small image
    P2 = P.copy(); P2[0, :] *= W / S.KITTI_W; P2[1, :] *= H / S.KITTI_H
    for kind, k in (("diamond", 5), ("rectangle", 3), ("cross", 7)):
        mask = S.structuring_element(kind, k)
        raw_ref = oracle.depth_project(pts, P2, W, H)
        ref = oracle.depth_inverse_dilation(raw_ref, mask)
        p = np.ascontiguousarray(pts, np.float32)
        raw = np.empty((H, W), np.float32); out = np.empty((H, W), np.float32)
        m = np.ascontiguousarray(mask, np.uint8)
        emu.emu_depth_dilate(L.ptr(p), p.shape[1], L.ptr(np.ascontiguousarray(P2.reshape(12))), W, H, L.ptr(m), m.shape[1], m.shape[0], 5.0, 200.0, 1.0,
                             L.ptr(raw), L.ptr(out))
        assert (raw.view(np.uint32) == raw_ref.view(np.uint32)).all()
        assert (out.view(np.uint32) == ref.view(np.uint32)).all(), kind
        assert (raw_ref > 0).sum() > 200 and (raw_ref[: H // 4] > 0).sum() == 0


def test_whole_extraction_pipeline_device_path(emu):
    """pyramid -> FAST -> compaction -> blur -> quad-tree -> describe through the real launchers on the emulator: keypoints and
    descriptors equal the oracle's ORBextractor::operator() bit for bit."""
    w, h = 260, 200
    img = S.make_image(81, w, h)
    prm = L.OrbParams(400, 1.2, 4, 12, 7)
    ok, od, _ = oracle.Extractor(400, 1.2, 4, 12, 7)(img)
    emu.emu_extract.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int]
    kps = np.empty(1024, oracle.KP_DTYPE); desc = np.empty((1024, 32), np.uint8)
    n = emu.emu_extract(C.byref(prm), L.ptr(img), w, h, img.strides[0], L.ptr(kps), L.ptr(desc), len(kps))
    assert n == len(ok) > 150
    for f in ok.dtype.names:
        assert (kps[:n][f].view(np.uint32) == ok[f].view(np.uint32)).all(), f
    assert (desc[:n] == od).all()


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_tlm_kernels_device_path(emu, seed):
    """The multi-CTA TrackLocalMap glue kernels (chain_kernels.cu: ordered compaction by 'publish and look back', the in-kernel grid
    barrier before the ring hand-over, self-cleaning slot arrays) against a serial restatement (tests/cuda_emu/tlm_check.cpp, which
    prints the first mismatches)."""
    assert emu.emu_tlm_check(seed) == 0

"""Stereo sequences on the device (System::TrackStereo -> GrabImageStereo -> stereo Frame constructor -> tracking): batched stereo frame
construction (both images of n pairs extracted as one batch, then the batched ComputeStereoMatches), the stereo sequence runner and the
stereo entry points' error handling, against the CPU oracle."""
import ctypes as C

import numpy as np
import pytest

import oracle
from oracle import stereo as ST
import tracking_data as TD
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S

pytestmark = pytest.mark.gpu

MB = float(np.float32(S.KITTI_BF) / np.float32(S.KITTI_FX))
MBF = float(S.KITTI_BF)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _same_frame(got, ref):
    k, d, dep, ur = got
    assert len(k) == len(ref["k"])
    for name in k.dtype.names:
        assert (_bits(k[name]) == _bits(ref["k"][name])).all(), name
    assert (d == ref["d"]).all()
    assert (_bits(dep) == _bits(ref["depth"])).all(), int((dep != ref["depth"]).sum())
    assert (_bits(ur) == _bits(ref["ur"])).all()


def test_stereo_frames_match_oracle():
    """upload (arrays and PNG bytes) + process + download of 4 pairs with the non-uniform disparity of stereo_pair vs the oracle's stereo
    Frame constructor, bit for bit; each pair also equals rgbl_stereo_matches on the same two slots of a batched extraction."""
    n = 4
    pairs = [S.stereo_pair(70 + p) for p in range(n)]
    lefts, rights = [p[0] for p in pairs], [p[1] for p in pairs]
    c = F.Context(S.KITTI_W, S.KITTI_H, 2000, max_batch=2 * n)
    try:
        b = F.StereoBatch(c, lefts, rights, pinned=False)
        b.upload()
        nk = b.process_resident(MB, MBF).copy()
        got = [tuple(np.array(a) for a in fr) for fr in b.download()]
        b.upload_png([S.encode_png(i) for i in lefts], [S.encode_png(i) for i in rights])
        b.process_resident(MB, MBF)
        got_png = [tuple(np.array(a) for a in fr) for fr in b.download()]
        ex = F.ORBextractor(2000, 1.2, 8, 12, 7, S.KITTI_W, S.KITTI_H, ctx=c)
        ex.extract_batch(lefts + rights)
        single = [F.stereo_matches_slots(ex, p, n + p, len(got[p][0]), MB, MBF) for p in range(n)]
    finally:
        c.close()
    exl, exr = oracle.Extractor(2000), oracle.Extractor(2000)
    for p in range(n):
        ref = ST.stereo_frame(exl, exr, lefts[p], rights[p], MB, MBF)
        assert nk[p] == len(ref["k"])
        _same_frame(got[p], ref)
        assert ((ref["depth"] > 0).sum() > 500) and (ref["depth"] < 0).any()
        for a, b2 in zip(got[p], got_png[p]):
            assert a.tobytes() == b2.tobytes()
        assert (_bits(single[p][0]) == _bits(got[p][2])).all() and (_bits(single[p][1]) == _bits(got[p][3])).all()


def _stereo_frames_oracle(seq, ts):
    exl, exr = oracle.Extractor(2000), oracle.Extractor(2000)
    return [ST.stereo_frame(exl, exr, seq.image(t), seq.right_image(t), MB, MBF) for t in ts], exl.scale_factors.copy()


def _run_stereo_sequence(seq, T, nB, K, resident):
    c = F.Context(S.KITTI_W, S.KITTI_H, 2000, max_batch=2 * T)
    try:
        r = F.SequenceRunner.stereo(c, MB, MBF, T, S.KITTI_W, S.KITTI_H, nB, pinned=False)
        for m in range(nB):
            ts = range(m * T, (m + 1) * T)
            r.set_batch(m, [seq.image(t) for t in ts], [seq.right_image(t) for t in ts])
            if resident:
                r.stage(m, m)
        cp = F.make_chain_params(seq.pose(0), *TD.CAM, th_last=7.0, continue_sequence=False, local_map_frames=K, th_local=1.0)
        o = r.run(cp, nB, first=0, resident_slots=nB if resident else 0, want_frames=True)
        return {k: np.array(v) for k, v in o.items()}
    finally:
        c.close()


@pytest.mark.parametrize("K", [2, 0])
def test_stereo_sequence_runner_matches_oracle_chain(K):
    """rgbl_track_sequence_stereo over three batches of one sequence, host and resident-staged mode (bitwise equal), vs oracle_chain2
    (th_last 7, th_local 1) on the oracle's stereo frames under the rule of test_rgbd_sequence_runner_matches_oracle_chain, and close to
    the synthetic truth."""
    T, nB = 5, 3
    seq = S.PlaneSequence(37, T * nB + 1)
    host = _run_stereo_sequence(seq, T, nB, K, False)
    res = _run_stereo_sequence(seq, T, nB, K, True)
    for k in host:
        assert host[k].tobytes() == res[k].tobytes(), k
    frames, sf = _stereo_frames_oracle(seq, range(T * nB))
    for t in range(T * nB):
        n = host["n_kp"][t]
        assert (_bits(host["depth"][t, :n]) == _bits(frames[t]["depth"])).all() and (host["desc"][t, :n] == frames[t]["d"]).all()
        assert (_bits(host["uright"][t, :n]) == _bits(frames[t]["ur"])).all()
    state = None
    in_sync, n_sync = True, 0
    for b in range(nB):
        rp, rnm, rni, rnl, rni1, state = TD.oracle_chain2(frames[b * T:(b + 1) * T], sf, seq.pose(0), K=K, th_last=7.0, th_local=1.0, state=state)
        for t in range(T):
            g = b * T + t
            if g == 0:
                continue
            if in_sync:
                assert host["n_matches"][g] == rnm[t] and host["n_local_matches"][g] == rnl[t] and host["n_inliers"][g] == rni[t], (b, t)
                assert np.abs(host["poses"][g] - rp[t]).max() < 2e-4, (b, t)
                n_sync += 1
                in_sync = np.abs(host["poses"][g] - rp[t]).max() <= 1e-7
            else:
                assert abs(int(host["n_matches"][g]) - int(rnm[t])) <= 6 and abs(int(host["n_local_matches"][g]) - int(rnl[t])) <= 10, (b, t)
                assert abs(int(host["n_inliers"][g]) - int(rni[t])) <= 10 and np.abs(host["poses"][g] - rp[t]).max() < 3e-3, (b, t)
        for t in range(T):
            assert abs(host["poses"][b * T + t, 4] - seq.pose(b * T + t)[4]) < 0.03, (b, t)
    # the first tracked frames agree in every count and within 1e-7 in the pose; with K = 0 the device's and the oracle's
    # PoseOptimization part in the last bits after two frames (th_last 7), after which the loose rule above applies
    assert n_sync >= 2, n_sync
    assert (host["n_inliers"][1:] > 150).all()


def _rgbl_and_rgbd(c, seq, T):
    """two chained RGB-L batches, then one RGB-D batch and its chain, on context c -> every output"""
    out = []
    prm = F.make_depth_params(bf=S.KITTI_BF)
    for b in range(2):
        ts = range(b * T, (b + 1) * T)
        rb = F.RgblBatch(c, [seq.image(t) for t in ts], [seq.cloud(t) for t in ts], seq.P, prm, pinned=False)
        rb.upload(); rb.process_resident()
        out.append([np.array(a) for fr in rb.download() for a in fr])
        rb.track_begin2(F.make_chain_params(seq.pose(0), *TD.CAM, continue_sequence=b > 0, local_map_frames=2))
        out.append(list(rb.track_end2().values()))
    db = F.RgbdBatch(c, [seq.image(t) for t in range(T)], [seq.depth16(t) for t in range(T)], pinned=False)
    db.upload(); db.process_resident(F.depth_map_factor(256), S.KITTI_BF)
    out.append([np.array(a) for fr in db.download() for a in fr])
    db.track_begin2(F.make_chain_params(seq.pose(0), *TD.CAM, local_map_frames=2))
    out.append(list(db.track_end2().values()))
    return out


def test_rgbl_and_rgbd_after_stereo_are_unchanged():
    """A context that ran stereo batches (stereo scratch allocated, chain state of a stereo sequence, slots [T, 2T) holding right images)
    gives bitwise the RGB-L and RGB-D results of a fresh context."""
    T = 4
    seq = S.PlaneSequence(42, 2 * T + 1)
    mk = lambda: F.Context(S.KITTI_W, S.KITTI_H, 2000, max_batch=2 * T, max_points=seq.cloud(0).shape[1])
    c = mk()
    try:
        ref = _rgbl_and_rgbd(c, seq, T)
    finally:
        c.close()
    c = mk()
    try:
        sb = F.StereoBatch(c, [seq.image(t) for t in range(T)], [seq.right_image(t) for t in range(T)], pinned=False)
        sb.upload(); sb.process_resident(MB, MBF)
        sb.track_begin2(F.make_chain_params(seq.pose(0), *TD.CAM, th_last=7.0, local_map_frames=2, th_local=1.0)); sb.track_end2()
        got = _rgbl_and_rgbd(c, seq, T)
    finally:
        c.close()
    for a, b in zip(ref, got):
        for p, q in zip(a, b):
            assert p.tobytes() == q.tobytes()


def _err(fn, code):
    with pytest.raises(L.RgblError) as e:
        fn()
    assert e.value.code == code, str(e.value)


def test_stereo_errors_leave_the_context_usable():
    T = 2
    seq = S.PlaneSequence(44, 2 * T)
    lefts, rights = [seq.image(t) for t in range(T)], [seq.right_image(t) for t in range(T)]
    clouds = [seq.cloud(t) for t in range(T)]
    c = F.Context(S.KITTI_W, S.KITTI_H, 1000, max_batch=2 * T, max_points=clouds[0].shape[1])
    lib, h = L.lib(), c.handle
    cp = F.make_chain_params(seq.pose(0), *TD.CAM, th_last=7.0, local_map_frames=2, th_local=1.0)
    try:
        # 2 n_pairs > max_batch (n_pairs itself fits)
        big = [seq.image(0)] * (T + 1)
        _err(lambda: F.StereoBatch(c, big, big, pinned=False).upload(), L.RGBL_E_INVALID)
        r3 = F.SequenceRunner.stereo(c, MB, MBF, T + 1, S.KITTI_W, S.KITTI_H, 1, pinned=False)
        r3.set_batch(0, big, big)
        _err(lambda: r3.run(cp, 1), L.RGBL_E_INVALID)
        _err(lambda: r3.stage(0, 0), L.RGBL_E_INVALID)
        # the process calls refuse the other kinds of upload
        sb = F.StereoBatch(c, lefts, rights, pinned=False)
        rb = F.RgblBatch(c, lefts, clouds, seq.P, F.make_depth_params(bf=S.KITTI_BF), pinned=False)
        db = F.RgbdBatch(c, lefts, [seq.depth16(t) for t in range(T)], pinned=False)
        assert lib.rgbl_resident_process_stereo(h, MB, MBF, None) == L.RGBL_E_INVALID                 # nothing uploaded
        rb.upload()
        assert lib.rgbl_resident_process_stereo(h, MB, MBF, None) == L.RGBL_E_INVALID
        db.upload()
        assert lib.rgbl_resident_process_stereo(h, MB, MBF, None) == L.RGBL_E_INVALID
        sb.upload()
        _err(rb.process_resident, L.RGBL_E_INVALID)
        _err(lambda: db.process_resident(F.depth_map_factor(256), S.KITTI_BF), L.RGBL_E_INVALID)
        assert lib.rgbl_resident_process_stereo(h, -1.0, MBF, None) == L.RGBL_E_INVALID
        # staged slots of the wrong kind, in both directions
        rs = F.SequenceRunner.stereo(c, MB, MBF, T, S.KITTI_W, S.KITTI_H, 1, pinned=False)
        rs.set_batch(0, lefts, rights); rs.stage(0, 0)
        rl = F.SequenceRunner(c, seq.P, F.make_depth_params(bf=S.KITTI_BF), T, S.KITTI_W, S.KITTI_H, clouds[0].shape[1], 1, pinned=False)
        rl.set_batch(0, lefts, clouds); rl.stage(1, 0)
        rd = F.SequenceRunner.rgbd(c, F.depth_map_factor(256), S.KITTI_BF, T, S.KITTI_W, S.KITTI_H, 1, pinned=False)
        rd.set_batch(0, lefts, [seq.depth16(t) for t in range(T)]); rd.stage(2, 0)
        _err(lambda: rl.run(cp, 1, first=0, resident_slots=1), L.RGBL_E_INVALID)          # slot 0 holds stereo pairs
        _err(lambda: rd.run(cp, 1, first=0, resident_slots=1), L.RGBL_E_INVALID)
        _err(lambda: rs.run(cp, 1, first=1, resident_slots=3), L.RGBL_E_INVALID)          # slot 1 holds RGB-L frames
        _err(lambda: rs.run(cp, 1, first=2, resident_slots=3), L.RGBL_E_INVALID)          # slot 2 holds RGB-D frames
        # point clouds given to the stereo runner; host mode without right images
        io = F.SequenceIO()
        io.n_batches, io.frames_per_batch, io.width, io.height, io.stride = 1, T, S.KITTI_W, S.KITTI_H, S.KITTI_W
        out = dict(poses=np.zeros((T, 7), np.float32), nm=np.zeros(T, np.int32), ni=np.zeros(T, np.int32))
        ga = (C.c_void_p * T)(*[i.ctypes.data for i in lefts]); ra = (C.c_void_p * T)(*[i.ctypes.data for i in rights])
        pa = (C.c_void_p * T)(*[clouds[0].ctypes.data] * T)
        io.gray = C.cast(ga, C.c_void_p); io.pts4xn = C.cast(pa, C.c_void_p)
        io.poses = out["poses"].ctypes.data; io.n_matches = out["nm"].ctypes.data; io.n_inliers = out["ni"].ctypes.data
        assert lib.rgbl_track_sequence_stereo(h, MB, MBF, C.byref(cp), C.byref(io), ra) == L.RGBL_E_INVALID
        io.pts4xn = None
        assert lib.rgbl_track_sequence_stereo(h, MB, MBF, C.byref(cp), C.byref(io), None) == L.RGBL_E_INVALID
        # a distorted camera: stereo needs rectified images
        c.set_camera_distortion(S.KITTI_FX, S.KITTI_FY, S.KITTI_CX, S.KITTI_CY, [-0.1, 0.01, 0.0, 0.0])
        _err(sb.upload, L.RGBL_E_UNSUPPORTED)
        _err(lambda: rs.run(cp, 1, first=0, resident_slots=1), L.RGBL_E_UNSUPPORTED)
        c.set_camera_distortion(S.KITTI_FX, S.KITTI_FY, S.KITTI_CX, S.KITTI_CY, [0.0, 0.0, 0.0, 0.0])
        # left and right PNGs of different sizes
        small = S.encode_png(np.ascontiguousarray(rights[0][:-2, :-4]))
        _err(lambda: sb.upload_png([S.encode_png(i) for i in lefts], [S.encode_png(rights[0]), small]), L.RGBL_E_INVALID)
        # calls while a chain is in flight
        sb.upload(); sb.process_resident(MB, MBF)
        sb.track_begin2(cp)
        _err(lambda: rs.run(cp, 1, first=0, resident_slots=1), L.RGBL_E_INVALID)
        d = np.empty(c.cap, np.float32)
        assert lib.rgbl_stereo_matches(h, 0, 1, MB, MBF, L.ptr(d), L.ptr(d), c.cap) == L.RGBL_E_INVALID
        o1 = sb.track_end2()
        assert (o1["n_inliers"][1:] > 100).all()
        # the context still works: every kind of slot through its own runner
        o = rs.run(cp, 1, first=0, resident_slots=3)
        assert (o["n_inliers"][1:] > 100).all() and o["poses"].tobytes() == o1["poses"].tobytes()
        o = rl.run(F.make_chain_params(seq.pose(0), *TD.CAM, local_map_frames=2), 1, first=1, resident_slots=3)
        assert (o["n_inliers"][1:] > 100).all()
        o = rd.run(F.make_chain_params(seq.pose(0), *TD.CAM, local_map_frames=2), 1, first=2, resident_slots=3)
        assert (o["n_inliers"][1:] > 100).all()
    finally:
        c.close()


"""Stereo rectification on the device (System::TrackStereo's cv::remap of both images before the stereo Frame constructor): batched
rectified stereo frames and the stereo sequence runner on raw pairs of a distorted EuRoC-like rig against the CPU oracle
(oracle/rectify.py), rectification switched off again, and the error cases."""
import ctypes as C

import numpy as np
import pytest

import oracle
from oracle import chain as CH
from oracle import rectify as RC
import test_rectify_cpu as RCPU
import tracking_data as TD
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S

pytestmark = pytest.mark.gpu

W, H, CAM, MB, MBF = RCPU.W, RCPU.H, RCPU.CAM, RCPU.MB, RCPU.MBF


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


def _rig_maps(seq):
    """M1l, M2l, M1r, M2r of a rig with R != I (rig_rotations)"""
    r1, r2 = RCPU.rig_rotations()
    return seq.rectification_maps(r1) + seq.rectification_maps(r2)


def _level0(c, n):
    out = []
    for f in range(n):
        img = np.empty((H, W), np.uint8)
        w, h = C.c_int(), C.c_int()
        F.check(L.lib().rgbl_orb_get_level(c.handle, f, 0, L.ptr(img), W, C.byref(w), C.byref(h)), c.handle)
        out.append(img)
    return out


def test_rectified_stereo_frames_match_oracle():
    """4 raw pairs in one batch, from arrays and from gray PNG bytes, rectified with R != I maps: level 0 of every left slot equals the
    oracle's remap; keypoints, descriptors, mvDepth and mvuRight equal rectified_stereo_frame bit for bit (the right images' remap is
    covered through mvDepth / mvuRight, whose SAD refinement reads the right pyramid)"""
    n = 4
    seq = RCPU.sequence(n=n + 1)
    lefts, rights = [seq.raw_left_image(t) for t in range(n)], [seq.raw_right_image(t) for t in range(n)]
    maps = _rig_maps(seq)
    c = F.Context(W, H, 2000, max_batch=2 * n)
    try:
        c.set_stereo_rectification(*maps)
        b = F.StereoBatch(c, lefts, rights, pinned=False)
        b.upload()
        nk = b.process_resident(MB, MBF).copy()
        got = [tuple(np.array(a) for a in fr) for fr in b.download()]
        lv = _level0(c, n)
        b.upload_png([S.encode_png(i) for i in lefts], [S.encode_png(i) for i in rights])
        b.process_resident(MB, MBF)
        got_png = [tuple(np.array(a) for a in fr) for fr in b.download()]
        lv_png = _level0(c, n)
    finally:
        c.close()
    exl, exr = oracle.Extractor(2000), oracle.Extractor(2000)
    for p in range(n):
        ref = RC.rectified_stereo_frame(exl, exr, lefts[p], rights[p], maps, MB, MBF)
        assert lv[p].tobytes() == ref["left"].tobytes() and lv_png[p].tobytes() == ref["left"].tobytes(), p
        assert nk[p] == len(ref["k"])
        _same_frame(got[p], ref)
        assert (ref["depth"] > 0).sum() > 50          # left and right rotated differently: fewer rows agree than in a true rig
        for a, b2 in zip(got[p], got_png[p]):
            assert a.tobytes() == b2.tobytes()


def _run(seq, T, nB, K, resident, maps):
    c = F.Context(W, H, 2000, max_batch=2 * T)
    try:
        if maps is not None:
            c.set_stereo_rectification(*maps)
        r = F.SequenceRunner.stereo(c, MB, MBF, T, W, H, nB, pinned=False)
        for m in range(nB):
            ts = range(m * T, (m + 1) * T)
            r.set_batch(m, [seq.raw_left_image(t) for t in ts], [seq.raw_right_image(t) for t in ts])
            if resident:
                r.stage(m, m)
        cp = F.make_chain_params(seq.pose(0), *CAM, th_last=7.0, continue_sequence=False, local_map_frames=K, th_local=1.0)
        o = r.run(cp, nB, first=0, resident_slots=nB if resident else 0, want_frames=True)
        return {k: np.array(v) for k, v in o.items()}
    finally:
        c.close()


@pytest.mark.parametrize("K", [2, 0])
def test_rectified_sequence_runner(K):
    """rgbl_track_sequence_stereo with rectification over three batches: host and resident mode give the same bits, the frames equal the
    oracle's rectified frames, the poses follow oracle_chain2 under the rule of test_gpu_stereo.py and stay within the CPU-established
    bounds, clearly below the errors of tracking the raw images without rectification"""
    T, nB = 5, 3
    seq = RCPU.sequence()
    maps = seq.rectification_maps() * 2
    host = _run(seq, T, nB, K, False, maps)
    res = _run(seq, T, nB, K, True, maps)
    for k in host:
        assert host[k].tobytes() == res[k].tobytes(), k
    exl, exr = oracle.Extractor(2000), oracle.Extractor(2000)
    frames = [RC.rectified_stereo_frame(exl, exr, seq.raw_left_image(t), seq.raw_right_image(t), maps, MB, MBF) for t in range(T * nB)]
    sf = exl.scale_factors.copy()
    for t in range(T * nB):
        n = host["n_kp"][t]
        assert (_bits(host["depth"][t, :n]) == _bits(frames[t]["depth"])).all() and (host["desc"][t, :n] == frames[t]["d"]).all()
        assert (_bits(host["uright"][t, :n]) == _bits(frames[t]["ur"])).all()
    state = None
    in_sync, n_sync = True, 0
    for b in range(nB):
        rp, rnm, rni, rnl, rni1, state = CH.oracle_chain2(frames[b * T:(b + 1) * T], sf, seq.pose(0), W, H, CAM, K=K, th_last=7.0, th_local=1.0,
                                                          state=state)
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
    assert n_sync >= 2, n_sync
    assert (host["n_inliers"][1:] > 100).all()
    e, dep = RCPU.errors(seq, host["poses"], [dict(depth=host["depth"][t, :host["n_kp"][t]]) for t in range(T * nB)])
    assert e[0] < RCPU.RECTIFIED_MAX_XY_ERR and e[1] < RCPU.RECTIFIED_MAX_XY_ERR and e[2] < RCPU.RECTIFIED_MAX_Z_ERR, e
    assert dep < RCPU.RECTIFIED_MAX_DEPTH_ERR, dep
    raw = _run(seq, T, nB, K, False, None)
    e_raw, dep_raw = RCPU.errors(seq, raw["poses"], [dict(depth=raw["depth"][t, :raw["n_kp"][t]]) for t in range(T * nB)])
    assert e_raw[2] > RCPU.RAW_MIN_Z_ERR and dep_raw > RCPU.RAW_MIN_DEPTH_ERR, (e_raw, dep_raw)


def _all_kinds(c, seq, T):
    """a stereo batch, two chained RGB-L batches and one RGB-D batch on context c (KITTI size, pinhole) -> every output"""
    out = []
    sb = F.StereoBatch(c, [seq.image(t) for t in range(T)], [seq.right_image(t) for t in range(T)], pinned=False)
    sb.upload(); sb.process_resident(float(np.float32(S.KITTI_BF) / np.float32(S.KITTI_FX)), S.KITTI_BF)
    out.append([np.array(a) for fr in sb.download() for a in fr])
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
    return out


def test_rectification_off_is_unchanged():
    """maps set and then cleared: stereo, RGB-L and RGB-D results are bitwise those of a fresh context"""
    T = 3
    seq = S.PlaneSequence(43, 2 * T + 1)
    mk = lambda: F.Context(S.KITTI_W, S.KITTI_H, 2000, max_batch=2 * T, max_points=seq.cloud(0).shape[1])
    c = mk()
    try:
        ref = _all_kinds(c, seq, T)
    finally:
        c.close()
    c = mk()
    try:
        maps = S.rectification_maps(S.KITTI_W, S.KITTI_H, TD.CAM[:4], S.EUROC_DIST)
        c.set_stereo_rectification(*(maps * 2))
        c.set_stereo_rectification(None, None, None, None)
        got = _all_kinds(c, seq, T)
    finally:
        c.close()
    for a, b in zip(ref, got):
        for p, q in zip(a, b):
            assert p.tobytes() == q.tobytes()


def _err(fn, code):
    with pytest.raises(L.RgblError) as e:
        fn()
    assert e.value.code == code, str(e.value)


def test_rectification_errors_leave_the_context_usable():
    T = 2
    seq = RCPU.sequence(n=T + 1)
    lefts, rights = [seq.raw_left_image(t) for t in range(T)], [seq.raw_right_image(t) for t in range(T)]
    maps = seq.rectification_maps() * 2
    c = F.Context(W, H, 1000, max_batch=2 * T)
    lib, h = L.lib(), c.handle
    try:
        m = [np.ascontiguousarray(a) for a in maps]
        p = [L.ptr(a) for a in m]
        assert lib.rgbl_set_stereo_rectification(h, p[0], None, p[2], p[3], W) == L.RGBL_E_INVALID          # partial NULLs
        assert lib.rgbl_set_stereo_rectification(h, p[0], p[1], p[2], p[3], W - 1) == L.RGBL_E_INVALID      # bad stride
        bad = m[2].copy(); bad[H - 1, W - 1] = np.nan
        assert lib.rgbl_set_stereo_rectification(h, p[0], p[1], L.ptr(bad), p[3], W) == L.RGBL_E_INVALID    # NaN
        # none of the above turned rectification on: the raw pair goes through the rectified path unremapped
        sb = F.StereoBatch(c, lefts, rights, pinned=False)
        sb.upload(); sb.process_resident(MB, MBF)
        assert (_bits(_level0(c, 1)[0]) == _bits(lefts[0])).all()
        c.set_stereo_rectification(*maps)
        # upload, then change the maps, then process: nothing uploaded
        sb.upload()
        c.set_stereo_rectification(*maps)
        _err(lambda: sb.process_resident(MB, MBF), L.RGBL_E_INVALID)
        sb.upload()
        c.set_stereo_rectification(None, None, None, None)
        _err(lambda: sb.process_resident(MB, MBF), L.RGBL_E_INVALID)
        c.set_stereo_rectification(*maps)
        # a colour PNG with rectification on
        col = [S.encode_png(S.colorize(i)) for i in lefts]
        _err(lambda: sb.upload_png(col, [S.encode_png(i) for i in rights]), L.RGBL_E_UNSUPPORTED)
        # a refused setting keeps the previous one, and the context still works
        assert lib.rgbl_set_stereo_rectification(h, p[0], p[1], L.ptr(bad), p[3], W) == L.RGBL_E_INVALID
        sb.upload_png([S.encode_png(i) for i in lefts], [S.encode_png(i) for i in rights])
        sb.process_resident(MB, MBF)
        exl, exr = oracle.Extractor(1000), oracle.Extractor(1000)
        ref = RC.rectified_stereo_frame(exl, exr, lefts[0], rights[0], maps, MB, MBF)
        _same_frame(tuple(np.array(a) for a in sb.download()[0]), ref)
    finally:
        c.close()

"""Distorted cameras on the device: Frame::UndistortKeyPoints and ComputeImageBounds (src/Frame.cc:837-899) through RGB-D and RGB-L frame
construction, the tracking chain and the RGB-D sequence runner, on a 640 x 480 sequence seen through TUM1's lens (k1..k3 != 0), against
the CPU oracle; and the default camera (k1 == 0) leaves every result as it was."""
import math

import numpy as np
import pytest

import oracle
from oracle import undistort as U
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S

pytestmark = pytest.mark.gpu

W, H = S.TUM_W, S.TUM_H
K4 = (S.TUM1_FX, S.TUM1_FY, S.TUM1_CX, S.TUM1_CY)
CAM = K4 + (S.TUM1_BF,)
DIST = S.TUM1_DIST
NFEAT = 1000
Z = 3.0                                      # a plane a few metres away, as indoors


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _seq(seed, n):
    return S.PlaneSequence(seed, n, Z=Z, W=W, H=H, cam=CAM, dist=DIST)


def _rgbd_inputs(seq, ts):
    return [seq.image(t) for t in ts], [seq.depth16(t, S.TUM_DEPTH_FACTOR, 0.05) for t in ts]


def _scale():
    return F.depth_map_factor(S.TUM_DEPTH_FACTOR)


def _ctx(T, dist=DIST, max_points=0):
    c = F.Context(W, H, NFEAT, max_batch=T, max_points=max_points)
    if dist is not None:
        c.set_camera_distortion(*K4, dist)
    return c


def _frames(b):
    return [tuple(np.array(a) for a in fr) for fr in b.download()], b.download_keys_un()


def test_rgbd_frames_match_oracle():
    """RGB-D frames of the distorted sequence, array and PNG uploads: mvKeys and descriptors equal a k1 = 0 run of the same images; mvKeysUn,
    mvDepth and mvuRight bit for bit against the oracle's RGB-D Frame constructor with the distortion; the bounds against the oracle."""
    T = 3
    seq = _seq(51, T)
    imgs, deps = _rgbd_inputs(seq, range(T))
    c = _ctx(T, None)
    try:
        assert list(c.set_camera_distortion(*K4, DIST)) == list(U.image_bounds(W, H, K4, DIST))
        b = F.RgbdBatch(c, imgs, deps, pinned=False)
        b.upload(); b.process_resident(_scale(), S.TUM1_BF)
        got, kun = _frames(b)
        b.upload_png([S.encode_png(i) for i in imgs], [S.encode_png16(d) for d in deps])
        b.process_resident(_scale(), S.TUM1_BF)
        got_png, kun_png = _frames(b)
    finally:
        c.close()
    c = _ctx(T, None)
    try:
        b = F.RgbdBatch(c, imgs, deps, pinned=False)
        b.upload(); b.process_resident(_scale(), S.TUM1_BF)
        plain, kun_plain = _frames(b)
    finally:
        c.close()
    ex = oracle.Extractor(NFEAT)
    for f in range(T):
        r = U.rgbd_frame(ex, imgs[f], deps[f], np.float32(_scale()), S.TUM1_BF, K4, DIST)
        k, d, dep, ur = got[f]
        assert k.tobytes() == plain[f][0].tobytes() and d.tobytes() == plain[f][1].tobytes()
        assert kun_plain[f].tobytes() == plain[f][0].tobytes()                       # k1 = 0: mvKeysUn == mvKeys
        assert k.tobytes() == r["k"].tobytes() and d.tobytes() == r["d"].tobytes()
        assert kun[f].tobytes() == r["kun"].tobytes()
        assert (_bits(dep) == _bits(r["depth"])).all() and (_bits(ur) == _bits(r["ur"])).all()
        assert (_bits(kun[f]["x"]) != _bits(k["x"])).mean() > 0.9                     # the lens moved the points
        assert (dep > 0).sum() > len(dep) // 2 and (dep < 0).any()
        assert (_bits(ur) != _bits(plain[f][3])).any()
        for a, b2 in zip(got[f] + (kun[f],), got_png[f] + (kun_png[f],)):
            assert a.tobytes() == b2.tobytes()


def test_rgbl_frames_match_oracle():
    """RGB-L frame construction (rgbl_resident_process) with the distortion: mvKeysUn from the device, mvDepth / mvuRight against the oracle
    DepthModule given mvKeys and mvKeysUn."""
    T = 2
    seq = _seq(52, T)
    prm = F.make_depth_params(min_dist=1.0, max_dist=50.0, bf=S.TUM1_BF)
    c = _ctx(T, DIST, seq.cloud(0).shape[1])
    try:
        rb = F.RgblBatch(c, [seq.image(t) for t in range(T)], [seq.cloud(t) for t in range(T)], seq.P, prm, pinned=False)
        rb.upload(); rb.process_resident()
        got, kun = _frames(rb)
    finally:
        c.close()
    ex = oracle.Extractor(NFEAT)
    mask = S.structuring_element("diamond", 5)
    for f in range(T):
        k, d, _ = ex(seq.image(f))
        rk = U.undistort_keypoints(k, K4, DIST)
        rdep, rur, _, _ = oracle.depth_from_pcd(seq.cloud(f), seq.P, W, H, mask, S.TUM1_BF, k, rk, 1.0, 50.0)
        assert got[f][0].tobytes() == k.tobytes() and got[f][1].tobytes() == d.tobytes()
        assert kun[f].tobytes() == rk.tobytes()
        assert (_bits(got[f][2]) == _bits(rdep)).all() and (_bits(got[f][3]) == _bits(rur)).all()
        assert (rdep > 0).sum() > 50


def _run_sequence(seq, T, nB, K, resident, dist=DIST):
    c = _ctx(T, dist)
    try:
        r = F.SequenceRunner.rgbd(c, _scale(), S.TUM1_BF, T, W, H, nB, pinned=False)
        for m in range(nB):
            imgs, deps = _rgbd_inputs(seq, range(m * T, (m + 1) * T))
            r.set_batch(m, imgs, deps)
            if resident:
                r.stage(m, m)
        cp = F.make_chain_params(seq.pose(0), *CAM, th_last=15.0, continue_sequence=False, local_map_frames=K, th_local=3.0)
        o = r.run(cp, nB, first=0, resident_slots=nB if resident else 0, want_frames=True)
        return {k: np.array(v) for k, v in o.items()}
    finally:
        c.close()


@pytest.mark.parametrize("K", [2, 0])
def test_rgbd_sequence_runner_distorted_matches_oracle_chain(K):
    """rgbl_track_sequence_rgbd on the distorted sequence, three batches, host and resident-staged (bitwise equal), against oracle_chain2 on
    the oracle's mvKeysUn frames with the undistorted image bounds (the rule of test_rgbd_sequence_runner_matches_oracle_chain), and close to
    the synthetic truth."""
    T, nB = 5, 3
    seq = _seq(56, T * nB + 1)
    host = _run_sequence(seq, T, nB, K, False)
    res = _run_sequence(seq, T, nB, K, True)
    for k in host:
        assert host[k].tobytes() == res[k].tobytes(), k
    ex = oracle.Extractor(NFEAT)
    imgs, deps = _rgbd_inputs(seq, range(T * nB))
    frames = []
    for t in range(T * nB):
        r = U.rgbd_frame(ex, imgs[t], deps[t], np.float32(_scale()), S.TUM1_BF, K4, DIST)
        frames.append(U.chain_frame(r))
        n = host["n_kp"][t]
        assert (_bits(host["depth"][t, :n]) == _bits(r["depth"])).all() and (_bits(host["uright"][t, :n]) == _bits(r["ur"])).all()
    bounds = U.image_bounds(W, H, K4, DIST)
    sf = ex.scale_factors.copy()
    state = None
    in_sync, n_sync = True, 0
    for b in range(nB):
        rp, rnm, rni, rnl, rni1, state = U.oracle_chain2(frames[b * T:(b + 1) * T], sf, seq.pose(0), W, H, CAM, bounds, K=K, state=state)
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
    err = np.abs(host["poses"][:, 4] - np.array([seq.pose(t)[4] for t in range(T * nB)]))
    assert err.max() < 0.01, err
    assert n_sync >= 3, n_sync
    assert (host["n_inliers"][1:] > 100).all()
    plain = _run_sequence(seq, T, nB, K, True, dist=None)
    err0 = np.abs(plain["poses"][:, 4] - np.array([seq.pose(t)[4] for t in range(T * nB)]))
    print(f"\nK={K}: max |x error| {err.max():.5f} m with the distortion, {err0.max():.5f} m with k1 = 0 "
          f"(inliers per frame {host['n_inliers'][1:].mean():.0f} vs {plain['n_inliers'][1:].mean():.0f})")


def _all_outputs(c, seq, T):
    """RGB-D frames + a chain, then RGB-L frames + a chain, on one context"""
    out = []
    imgs, deps = _rgbd_inputs(seq, range(T))
    b = F.RgbdBatch(c, imgs, deps, pinned=False)
    b.upload(); b.process_resident(_scale(), S.TUM1_BF)
    fr, kun = _frames(b)
    b.track_begin2(F.make_chain_params(seq.pose(0), *CAM, local_map_frames=2))
    out += [x for f in fr for x in f] + kun + list(b.track_end2().values())
    prm = F.make_depth_params(min_dist=1.0, max_dist=50.0, bf=S.TUM1_BF)
    rb = F.RgblBatch(c, imgs, [seq.cloud(t) for t in range(T)], seq.P, prm, pinned=False)
    rb.upload(); rb.process_resident()
    fr, kun = _frames(rb)
    rb.track_begin2(F.make_chain_params(seq.pose(0), *CAM, local_map_frames=2))
    out += [x for f in fr for x in f] + kun + list(rb.track_end2().values())
    return [np.asarray(a).tobytes() for a in out]


def test_default_camera_changes_nothing():
    """k1 = 0 with non-zero k2..k3 (the reference's early return) gives the results of a context whose camera was never set, and so does a
    context set to TUM1, used, and set back to k1 = 0 (the cached chain graph is re-captured with the image bounds)."""
    T = 4
    seq = _seq(57, T)
    npts = seq.cloud(0).shape[1]
    ref_c = _ctx(T, None, npts)
    try:
        ref = _all_outputs(ref_c, seq, T)
    finally:
        ref_c.close()
    k1zero = np.array([0.0, -0.95, 0.004, 0.002, 1.1], np.float32)
    c = _ctx(T, None, npts)
    try:
        assert list(c.set_camera_distortion(*K4, k1zero)) == [0, W, 0, H]
        assert _all_outputs(c, seq, T) == ref
    finally:
        c.close()
    c = _ctx(T, DIST, npts)
    try:
        dist_out = _all_outputs(c, seq, T)
        assert dist_out != ref
        c.set_camera_distortion(*K4, k1zero[:4])
        assert _all_outputs(c, seq, T) == ref
    finally:
        c.close()


def test_distortion_errors_leave_the_context_usable():
    T = 2
    seq = _seq(58, T)
    imgs, deps = _rgbd_inputs(seq, range(T))
    c = _ctx(T, None)
    lib, h = L.lib(), c.handle
    b6 = np.zeros(4, np.float32)

    def setc(fx, fy, cx, cy, dist):
        d = np.ascontiguousarray(dist, np.float32)
        return lib.rgbl_set_camera_distortion(h, fx, fy, cx, cy, L.ptr(d), len(d), L.ptr(b6))
    try:
        good = c.set_camera_distortion(*K4, DIST)
        for n in (3, 6):
            assert setc(*K4, np.resize(DIST, n)) == L.RGBL_E_INVALID, n
        assert setc(*K4, [math.nan, 0, 0, 0]) == L.RGBL_E_INVALID
        assert setc(math.nan, K4[1], K4[2], K4[3], DIST) == L.RGBL_E_INVALID
        assert setc(0.0, K4[1], K4[2], K4[3], DIST) == L.RGBL_E_INVALID
        assert setc(K4[0], -1.0, K4[2], K4[3], DIST) == L.RGBL_E_INVALID
        assert lib.rgbl_set_camera_distortion(h, *K4, None, 5, None) == L.RGBL_E_INVALID
        b = F.RgbdBatch(c, imgs, deps, pinned=False)
        b.upload(); b.process_resident(_scale(), S.TUM1_BF)
        b.track_begin2(F.make_chain_params(seq.pose(0), *CAM, local_map_frames=2))
        assert setc(*K4, np.zeros(4)) == L.RGBL_E_INVALID                       # a chain is in flight
        o = b.track_end2()
        assert (o["n_inliers"][1:] > 100).all()
        # the failed calls changed nothing: the context still undistorts with TUM1
        _, kun = _frames(b)
        r = U.rgbd_frame(oracle.Extractor(NFEAT), imgs[0], deps[0], np.float32(_scale()), S.TUM1_BF, K4, DIST)
        assert kun[0].tobytes() == r["kun"].tobytes()
        assert setc(*K4, DIST) == 0 and b6.tobytes() == good.tobytes()
    finally:
        c.close()

"""RGB-D sequences on the device (System::TrackRGBD -> GrabImageRGBD -> RGB-D Frame constructor -> tracking): the 16-bit depth PNG
decode, RGB-D frame construction (extraction + ComputeStereoFromRGBD on the uint16 depth planes scaled like GrabImageRGBD's
convertTo) and the RGB-D sequence runner, against the CPU oracle."""
import ctypes as C

import numpy as np
import pytest

import oracle
from oracle import rgbd as R
import tracking_data as TD
from orb_slam3_rgbl_b200 import _lib as L
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


@pytest.mark.parametrize("W,H", [(S.KITTI_W, S.KITTI_H), (1920, 1080), (333, 1100)])
def test_decode_png_depth16_matches_oracle(W, H):
    rng = np.random.default_rng(W + H)
    seq = S.PlaneSequence(4, 2, W=W, H=H)
    imgs = [seq.depth16(0, 256.0, 0.05), rng.integers(0, 65536, (H, W)).astype(np.uint16)]
    pngs = [S.encode_png16(imgs[0]), S.encode_png16(imgs[1], rng.integers(0, 5, H), 20000)]
    if (W, H) == (333, 1100):
        pngs += [S.encode_png16(imgs[1], np.full(H, ft)) for ft in range(5)]
    c = F.Context(W, H, 1000, max_batch=len(pngs))
    try:
        got = F.decode_png_depth16(c, pngs)
    finally:
        c.close()
    for g, png in zip(got, pngs):
        assert (g == R.png_decode_depth16(png)).all()


def _rgbd_inputs(seq, ts, factor):
    deps = [seq.depth16(t, factor, 0.05) for t in ts]
    if factor == 1:          # the whole uint16 range (holes kept)
        deps = [np.where(d > 0, np.random.default_rng(t).integers(1, 65536, d.shape), 0).astype(np.uint16) for t, d in zip(ts, deps)]
    return [seq.image(t) for t in ts], deps


@pytest.mark.parametrize("factor", [256, 5000, 1])
def test_rgbd_frames_match_oracle(factor):
    """upload + process + download of RGB-D frames vs the oracle's RGB-D Frame constructor: keypoints, descriptors, mvDepth, mvuRight
    bit for bit (also against the reference's own ComputeStereoFromRGBD when it is built), and the PNG upload gives the same bits."""
    T = 3
    seq = S.PlaneSequence(21, T)
    imgs, deps = _rgbd_inputs(seq, range(T), factor)
    scale = F.depth_map_factor(factor)
    c = F.Context(S.KITTI_W, S.KITTI_H, 2000, max_batch=T)
    try:
        b = F.RgbdBatch(c, imgs, deps, pinned=False)
        b.upload(); b.process_resident(scale, S.KITTI_BF)
        got = [tuple(np.array(a) for a in fr) for fr in b.download()]
        b.upload_png([S.encode_png(i) for i in imgs], [S.encode_png16(d) for d in deps])
        b.process_resident(scale, S.KITTI_BF)
        got_png = [tuple(np.array(a) for a in fr) for fr in b.download()]
    finally:
        c.close()
    ex = oracle.Extractor(2000)
    ref_tr = oracle.ref_tracking()
    for f in range(T):
        r = R.rgbd_frame(ex, imgs[f], deps[f], np.float32(scale), S.KITTI_BF)
        k, d, dep, ur = got[f]
        assert len(k) == len(r["k"])
        for name in k.dtype.names:
            assert (_bits(k[name]) == _bits(r["k"][name])).all(), name
        assert (d == r["d"]).all()
        assert (_bits(dep) == _bits(r["depth"])).all() and (_bits(ur) == _bits(r["ur"])).all()
        assert (dep > 0).sum() > len(dep) // 2 and (dep < 0).any()
        if ref_tr is not None:
            xy = np.stack([k["x"], k["y"]], 1)
            rd, ru = oracle.ref_stereo_from_rgbd(xy, xy, R.depth_scale(deps[f], scale), S.KITTI_BF)
            assert (_bits(dep) == _bits(rd)).all() and (_bits(ur) == _bits(ru)).all()
        for a, b2 in zip(got[f], got_png[f]):
            assert a.tobytes() == b2.tobytes()


def _run_rgbd_sequence(seq, T, nB, K, resident, factor=256.0):
    c = F.Context(S.KITTI_W, S.KITTI_H, 2000, max_batch=T)
    try:
        r = F.SequenceRunner.rgbd(c, F.depth_map_factor(factor), S.KITTI_BF, T, S.KITTI_W, S.KITTI_H, nB, pinned=False)
        for m in range(nB):
            imgs, deps = _rgbd_inputs(seq, range(m * T, (m + 1) * T), factor)
            r.set_batch(m, imgs, deps)
            if resident:
                r.stage(m, m)
        cp = F.make_chain_params(seq.pose(0), *TD.CAM, th_last=15.0, continue_sequence=False, local_map_frames=K, th_local=3.0)
        o = r.run(cp, nB, first=0, resident_slots=nB if resident else 0, want_frames=True)
        return {k: np.array(v) for k, v in o.items()}
    finally:
        c.close()


@pytest.mark.parametrize("K", [2, 0])
def test_rgbd_sequence_runner_matches_oracle_chain(K):
    """rgbl_track_sequence_rgbd over three batches of one sequence, host and resident-staged mode (bitwise equal), vs oracle_chain2 on
    the oracle's RGB-D frames under the rule of test_full_tracking_chain_continuous_sequence, and close to the synthetic truth."""
    T, nB = 5, 3
    seq = S.PlaneSequence(36, T * nB + 1)
    host = _run_rgbd_sequence(seq, T, nB, K, False)
    res = _run_rgbd_sequence(seq, T, nB, K, True)
    for k in host:
        assert host[k].tobytes() == res[k].tobytes(), k
    ex = oracle.Extractor(2000)
    imgs, deps = _rgbd_inputs(seq, range(T * nB), 256)
    frames = [R.rgbd_frame(ex, imgs[t], deps[t], np.float32(F.depth_map_factor(256)), S.KITTI_BF) for t in range(T * nB)]
    sf = ex.scale_factors.copy()
    for t in range(T * nB):
        n = host["n_kp"][t]
        assert (_bits(host["depth"][t, :n]) == _bits(frames[t]["depth"])).all() and (host["desc"][t, :n] == frames[t]["d"]).all()
    state = None
    in_sync, n_sync = True, 0
    for b in range(nB):
        rp, rnm, rni, rnl, rni1, state = TD.oracle_chain2(frames[b * T:(b + 1) * T], sf, seq.pose(0), K=K, state=state)
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
            assert abs(host["poses"][b * T + t, 4] - seq.pose(b * T + t)[4]) < 0.03
    assert n_sync >= 3, n_sync
    assert (host["n_inliers"][1:] > 150).all()


def _rgbl_chain(c, seq, T):
    prm = F.make_depth_params(bf=S.KITTI_BF)
    out = []
    for b in range(2):
        ts = range(b * T, (b + 1) * T)
        rb = F.RgblBatch(c, [seq.image(t) for t in ts], [seq.cloud(t) for t in ts], seq.P, prm, pinned=False)
        rb.upload(); rb.process_resident()
        frames = [tuple(np.array(a) for a in fr) for fr in rb.download()]
        rb.track_begin2(F.make_chain_params(seq.pose(0), *TD.CAM, continue_sequence=b > 0, local_map_frames=2))
        out.append((frames, rb.track_end2()))
    return out


def test_rgbl_after_rgbd_is_unchanged():
    """A context that ran RGB-D batches (depth planes allocated, chain state of an RGB-D sequence) gives bitwise the RGB-L results of a
    fresh context."""
    T = 4
    seq = S.PlaneSequence(41, 2 * T + 1)
    mk = lambda: F.Context(S.KITTI_W, S.KITTI_H, 2000, max_batch=T, max_points=seq.cloud(0).shape[1])
    c = mk()
    try:
        ref = _rgbl_chain(c, seq, T)
    finally:
        c.close()
    c = mk()
    try:
        imgs, deps = _rgbd_inputs(seq, range(T), 256)
        b = F.RgbdBatch(c, imgs, deps, pinned=False)
        b.upload(); b.process_resident(F.depth_map_factor(256), S.KITTI_BF)
        b.track_begin2(F.make_chain_params(seq.pose(0), *TD.CAM, local_map_frames=2)); b.track_end2()
        got = _rgbl_chain(c, seq, T)
    finally:
        c.close()
    for (fa, ta), (fb, tb) in zip(ref, got):
        for x, y in zip(fa, fb):
            for p, q in zip(x, y):
                assert p.tobytes() == q.tobytes()
        for k in ta:
            assert ta[k].tobytes() == tb[k].tobytes(), k


def test_rgbd_errors_leave_the_context_usable():
    T = 2
    seq = S.PlaneSequence(43, T)
    imgs, deps = _rgbd_inputs(seq, range(T), 256)
    c = F.Context(S.KITTI_W, S.KITTI_H, 1000, max_batch=T, max_points=seq.cloud(0).shape[1])
    scale, bf = F.depth_map_factor(256), S.KITTI_BF
    lib, h = L.lib(), c.handle
    try:
        assert lib.rgbl_resident_process_rgbd(h, scale, bf, None) == L.RGBL_E_INVALID           # nothing uploaded
        rb = F.RgblBatch(c, imgs, [seq.cloud(t) for t in range(T)], seq.P, F.make_depth_params(bf=bf), pinned=False)
        rb.upload()
        assert lib.rgbl_resident_process_rgbd(h, scale, bf, None) == L.RGBL_E_INVALID           # RGB-L frames uploaded
        # a staged slot of the wrong kind, for both runners
        rl = F.SequenceRunner(c, seq.P, F.make_depth_params(bf=bf), T, S.KITTI_W, S.KITTI_H, seq.cloud(0).shape[1], 1, pinned=False)
        rl.set_batch(0, imgs, [seq.cloud(t) for t in range(T)]); rl.stage(0, 0)
        rd = F.SequenceRunner.rgbd(c, scale, bf, T, S.KITTI_W, S.KITTI_H, 1, pinned=False)
        rd.set_batch(0, imgs, deps); rd.stage(1, 0)
        cp = F.make_chain_params(seq.pose(0), *TD.CAM, local_map_frames=2)
        with pytest.raises(L.RgblError) as e:
            rd.run(cp, 1, first=0, resident_slots=1)                     # slot 0 holds RGB-L frames
        assert e.value.code == L.RGBL_E_INVALID
        with pytest.raises(L.RgblError) as e:
            rl.run(cp, 1, first=1, resident_slots=2)                     # slot 1 holds RGB-D frames
        assert e.value.code == L.RGBL_E_INVALID
        # pts4xn given to the RGB-D runner
        out = dict(poses=np.zeros((T, 7), np.float32), nm=np.zeros(T, np.int32), ni=np.zeros(T, np.int32))
        io = F.SequenceIO()
        io.n_batches, io.frames_per_batch, io.width, io.height, io.stride = 1, T, S.KITTI_W, S.KITTI_H, S.KITTI_W
        ga = (C.c_void_p * T)(*[i.ctypes.data for i in imgs]); pa = (C.c_void_p * T)(*[seq.cloud(0).ctypes.data] * T)
        da = (C.c_void_p * T)(*[d.ctypes.data for d in deps])
        io.gray = C.cast(ga, C.c_void_p); io.pts4xn = C.cast(pa, C.c_void_p)
        io.poses = out["poses"].ctypes.data; io.n_matches = out["nm"].ctypes.data; io.n_inliers = out["ni"].ctypes.data
        assert lib.rgbl_track_sequence_rgbd(h, scale, bf, C.byref(cp), C.byref(io), da, S.KITTI_W) == L.RGBL_E_INVALID
        # a depth PNG that is not 16-bit gray
        for png in (S.encode_png(imgs[0]), S.encode_png16(np.stack([deps[0]] * 3, -1))):
            with pytest.raises(L.RgblError) as e:
                F.decode_png_depth16(c, [png, png])
            assert e.value.code == L.RGBL_E_UNSUPPORTED
        # the context still works: the RGB-D slot through the RGB-D runner, the RGB-L slot through the RGB-L runner
        o = rd.run(cp, 1, first=1, resident_slots=2)
        assert (o["n_inliers"][1:] > 100).all()
        o = rl.run(cp, 1, first=0, resident_slots=2)
        assert (o["n_inliers"][1:] > 100).all()
    finally:
        c.close()

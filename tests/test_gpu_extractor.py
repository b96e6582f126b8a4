"""GPU parity: CUDA ORB extractor (through the C ABI) vs the CPU oracle, stage by stage and end to end.
Bar: bit-exact (integer/byte/index work; angles are float32 results of identical operation sequences)."""
import numpy as np
import pytest

import oracle
from orb_slam3_rgbl_b200 import frontend as F
from orb_slam3_rgbl_b200 import synthetic as S

pytestmark = pytest.mark.gpu


def _cmp_kps(a, b):
    assert len(a) == len(b), f"keypoint count {len(a)} vs oracle {len(b)}"
    bad = {f: int((a[f] != b[f]).sum()) for f in a.dtype.names}
    assert not any(bad.values()), f"keypoint field mismatches: {bad}"


@pytest.fixture(scope="module")
def kitti_ctx():
    ex = F.ORBextractor(2000, 1.2, 8, 12, 7, S.KITTI_W, S.KITTI_H, max_batch=4)
    yield ex
    ex.ctx.close()


@pytest.mark.parametrize("seed", [0, 11])
def test_stages_and_keypoints_kitti(kitti_ctx, seed, report_dir):
    img = S.make_image(seed)
    ref = oracle.Extractor(2000)
    rk, rd, rmono = ref(img)
    mono, k, d = kitti_ctx(img)
    lines = []
    for l in range(8):
        a, b = kitti_ctx.level_image(l), ref.level_image(l)
        assert a.shape == b.shape
        lines.append(f"level {l}: pyramid mismatches {(a != b).sum()}")
        assert (a == b).all(), lines[-1]
        ab, bb = kitti_ctx.blurred_level(l), oracle.gaussian_blur7(b)
        lines.append(f"level {l}: blur mismatches {(ab != bb).sum()}")
        assert (ab == bb).all(), lines[-1]
        ca, cb = kitti_ctx.level_candidates(l), ref.level_candidates(l)
        lines.append(f"level {l}: candidates {len(ca)} vs {len(cb)}")
        assert ca.shape == cb.shape and (ca == cb).all(), lines[-1]
    (report_dir / f"extractor_stage_report_{seed}.txt").write_text("\n".join(lines))
    _cmp_kps(k, rk)
    assert (d == rd).all(), f"descriptor rows differing: {(d != rd).any(axis=1).sum()}"
    assert mono == rmono


def test_host_and_device_quadtree_agree(kitti_ctx):
    img = S.make_image(41)
    rk, rd, _ = oracle.Extractor(2000)(img)
    try:
        for host in (True, False):
            kitti_ctx.ctx.set_host_quadtree(host)
            mono, k, d = kitti_ctx(img)
            _cmp_kps(k, rk)
            assert (d == rd).all()
    finally:
        kitti_ctx.ctx.set_host_quadtree(False)


def test_batch_equals_single(kitti_ctx):
    imgs = [S.make_image(s) for s in (21, 22, 23)]
    outs = kitti_ctx.extract_batch(imgs)
    ref = oracle.Extractor(2000)
    for img, (k, d) in zip(imgs, outs):
        rk, rd, _ = ref(img)
        _cmp_kps(k, rk)
        assert (d == rd).all()


def test_padded_pyramid_matches_reflect101(kitti_ctx):
    img = S.make_image(3)
    kitti_ctx(img)
    ref = oracle.Extractor(2000); ref(img)
    for l in (0, 3, 7):
        p = kitti_ctx.image_pyramid_padded(l)
        r = np.pad(ref.level_image(l), 19, mode="reflect")       # numpy 'reflect' == BORDER_REFLECT_101
        assert p.shape == r.shape and (p == r).all()


@pytest.mark.parametrize("w,h,nf", [(640, 480, 1000), (752, 480, 1200), (1920, 1080, 4000)])
def test_other_sizes(w, h, nf):
    img = S.make_image(7, w, h)
    ex = F.ORBextractor(nf, 1.2, 8, 12, 7, w, h)
    try:
        mono, k, d = ex(img)
    finally:
        ex.ctx.close()
    rk, rd, _ = oracle.Extractor(nf)(img)
    _cmp_kps(k, rk)
    assert (d == rd).all()


@pytest.mark.parametrize("scale,levels,nf", [(1.5, 5, 1500), (1.1, 8, 2000), (1.35, 6, 1000), (1.6, 4, 800)])
def test_other_scale_factors(scale, levels, nf):
    """Settings other than the KITTI yaml: the staged-tile resize kernel serves level ratios up to ~1.35, larger ones take the
    gather kernel; both must stay bit-exact with the oracle (pyramid, keypoints, descriptors)."""
    img = S.make_image(5, S.KITTI_W, S.KITTI_H)
    ex = F.ORBextractor(nf, scale, levels, 12, 7, S.KITTI_W, S.KITTI_H)
    try:
        mono, k, d = ex(img)
        pyr = [ex.level_image(l) for l in range(levels)]
    finally:
        ex.ctx.close()
    ref = oracle.Extractor(nf, scale, levels)
    rk, rd, _ = ref(img)
    for l in range(levels):
        assert np.array_equal(pyr[l], ref.level_image(l)), f"level {l} differs"
    _cmp_kps(k, rk)
    assert (d == rd).all()


def test_flat_image_gives_no_keypoints():
    img = np.full((S.KITTI_H, S.KITTI_W), 100, np.uint8)
    ex = F.ORBextractor(1000, 1.2, 8, 12, 7, S.KITTI_W, S.KITTI_H)
    try:
        mono, k, d = ex(img)
    finally:
        ex.ctx.close()
    assert mono == 0 and len(k) == 0 and d.shape == (0, 32)


def test_empty_image_returns_minus_one(kitti_ctx):
    mono, k, d = kitti_ctx(np.empty((0, 0), np.uint8))
    assert mono == -1


def test_low_texture_uses_min_threshold():
    # faint texture: most cells fall back to minThFAST=7 (src/ORBextractor.cc:843-846)
    rng = np.random.default_rng(5)
    img = (100 + 6 * rng.standard_normal((S.KITTI_H, S.KITTI_W))).clip(0, 255).astype(np.uint8)
    ex = F.ORBextractor(1000, 1.2, 8, 12, 7, S.KITTI_W, S.KITTI_H)
    try:
        mono, k, d = ex(img)
    finally:
        ex.ctx.close()
    rk, rd, _ = oracle.Extractor(1000)(img)
    _cmp_kps(k, rk)
    assert (d == rd).all()


def test_compute_stereo_matches():
    """Frame::ComputeStereoMatches on a synthetic rectified pair (uniform 5 px disparity): bit-exact mvDepth / mvuRight."""
    tex = S.make_image(77, S.KITTI_W + 40, S.KITTI_H)
    left = np.ascontiguousarray(tex[:, 10:10 + S.KITTI_W]); right = np.ascontiguousarray(tex[:, 15:15 + S.KITTI_W])
    el, er = oracle.Extractor(2000), oracle.Extractor(2000)
    kl, dl, _ = el(left); kr, dr, _ = er(right)
    mb = np.float32(S.KITTI_BF) / np.float32(S.KITTI_FX); mbf = np.float32(S.KITTI_BF)
    rd, ru = oracle.stereo_matches(kl, dl, kr, dr, el, er, mb, mbf)
    ex = F.ORBextractor(2000, 1.2, 8, 12, 7, S.KITTI_W, S.KITTI_H, max_batch=2)
    try:
        (gkl, gdl), (gkr, gdr), gd, gu = F.compute_stereo_matches(ex, (left, right), float(mb), float(mbf))
    finally:
        ex.ctx.close()
    _cmp_kps(gkl, kl); _cmp_kps(gkr, kr)
    assert (gd == rd).all() and (gu == ru).all(), f"{(gd != rd).sum()} depths differ"
    ok = rd > 0
    assert ok.sum() > 800 and abs(np.median(kl["x"][ok] - ru[ok]) - 5.0) < 0.05


@pytest.mark.parametrize("W,H,scale,nlevels", [(S.KITTI_W, S.KITTI_H, 1.2, 8), (641, 481, 1.2, 8), (752, 480, 1.44, 5), (515, 389, 2.0, 3), (1920, 1080, 1.2, 8)])
def test_fused_tma_level_kernel_equals_oracle_and_two_pass_kernels(W, H, scale, nlevels, monkeypatch):
    """level_tma_kernels.cu (TMA box loads + IDP4A/IDP2A blur + resize from the same tile) against the oracle's cv::resize /
    cv::GaussianBlur restatements and against the two-pass kernels (RGBL_LEVEL_TMA=0), every level, every frame slot of a batch:
    sizes with partial edge tiles in both directions, widths that are not multiples of 4, other level ratios."""
    imgs = [S.make_image(60 + i, W, H, n_rects=150) for i in range(3)]
    ref = oracle.Extractor(1000, scale, nlevels)
    outs = {}
    for tma in ("1", "0"):
        monkeypatch.setenv("RGBL_LEVEL_TMA", tma)
        ex = F.ORBextractor(1000, scale, nlevels, 12, 7, W, H, max_batch=3)
        try:
            res = ex.extract_batch(imgs)
            outs[tma] = [[(ex.level_image(l, f), ex.blurred_level(l, f)) for l in range(nlevels)] for f in range(3)]
            for img, (k, d) in zip(imgs, res):
                rk, rd, _ = ref(img)
                _cmp_kps(k, rk)
                assert (d == rd).all()
        finally:
            ex.ctx.close()
    for f in range(3):
        ref(imgs[f])
        for l in range(nlevels):
            a, ab = outs["1"][f][l]
            b, bb = outs["0"][f][l]
            r = ref.level_image(l)
            assert a.shape == r.shape and (a == r).all(), f"frame {f} level {l}: pyramid mismatches {(a != r).sum()}"
            assert (ab == oracle.gaussian_blur7(r)).all(), f"frame {f} level {l}: blur mismatches {(ab != oracle.gaussian_blur7(r)).sum()}"
            assert (a == b).all() and (ab == bb).all()


def test_two_pass_levels_and_host_quadtree_frames_equal_the_oracle(monkeypatch):
    """The paths besides the defaults that a context can take: the two-pass pyramid + blur (RGBL_LEVEL_TMA=0, also the path of level
    ratios the fused tile kernel cannot hold) and the host quad-tree (rgbl_set_host_quadtree, also the path of level geometries the device
    quad-tree cannot hold).  One RGB-L frame construction with each equals the oracle bit for bit, like the default kernels do."""
    W, H = S.KITTI_W, S.KITTI_H
    img = S.make_image(77, W, H)
    pts = S.make_pointcloud(77)
    P = S.lidar_projection_matrix()
    rk, rd, _ = oracle.Extractor(2000)(img)
    rdep, rur, _, _ = oracle.depth_from_pcd(pts, P, W, H, S.structuring_element("diamond", 5), S.KITTI_BF, rk, rk)
    for level_tma, host_quadtree in (("0", False), ("1", True)):
        monkeypatch.setenv("RGBL_LEVEL_TMA", level_tma)                # read by rgbl_create
        ctx = F.Context(W, H, 2000, max_batch=1, max_points=pts.shape[1])
        try:
            ctx.set_host_quadtree(host_quadtree)
            (k, d, dep, ur), = F.frame_rgbl_batch(ctx, [img], [pts], P, F.make_depth_params(bf=S.KITTI_BF))
        finally:
            ctx.close()
        _cmp_kps(k, rk)
        assert (d == rd).all() and (dep == rdep).all() and (ur == rur).all(), (level_tma, host_quadtree)

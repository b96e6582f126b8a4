"""Host-side mirror of the reference's hot-path classes on top of the C ABI.

Names and argument meaning follow the reference so the parity tests read like reference usage:
  ORBextractor  <- include/ORBextractor.h:45-108  (operator() -> __call__)
  DepthModule   <- include/DepthModule.h:30-164   (CalculateDepthFromPcd, mvDepth, mvuRight, ...)
All compute happens in librgbl_b200.so on the GPU; this file only marshals numpy buffers.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib as L
from ._lib import KP_DTYPE, DepthParams, OrbParams, check, lib, ptr


class Context:
    """One rgbl_ctx: fixed image size, batch capacity and ORB parameters, bound to one CUDA device."""

    def __init__(self, width: int, height: int, nfeatures=2000, scale_factor=1.2, nlevels=8, ini_th=12, min_th=7,
                 max_batch=1, max_points=0, max_candidates=0, device=0):
        self.orb = OrbParams(nfeatures, scale_factor, nlevels, ini_th, min_th)
        self.cfg = L.Config(device, width, height, max_batch, max_points, max_candidates, self.orb)
        self.handle = C.c_void_p()
        rc = lib().rgbl_create(C.byref(self.cfg), C.byref(self.handle))
        if rc != 0:
            msg = lib().rgbl_last_error(None)
            raise L.RgblError(rc, msg.decode() if msg else "rgbl_create failed")
        self.width, self.height, self.nlevels, self.nfeatures = width, height, nlevels, nfeatures
        self.max_batch = max_batch
        self.cap = lib().rgbl_keypoint_capacity(self.handle)

    # ---- profiling / timing (rgbl_profile_*, rgbl_timer_*) ----
    def profile_enable(self, on=True):
        check(lib().rgbl_profile_enable(self.handle, int(on)), self.handle)

    def profile_reset(self):
        check(lib().rgbl_profile_reset(self.handle), self.handle)

    def profile_read(self) -> dict:
        out = {}
        for s in range(lib().rgbl_profile_num_stages()):
            ms, nl, nc = C.c_double(), C.c_int64(), C.c_int64()
            check(lib().rgbl_profile_read(self.handle, s, C.byref(ms), C.byref(nl), C.byref(nc)), self.handle)
            out[lib().rgbl_profile_stage_name(s).decode()] = dict(ms=ms.value, launches=nl.value, calls=nc.value)
        nl, hq = C.c_int64(), C.c_double()
        check(lib().rgbl_profile_totals(self.handle, C.byref(nl), C.byref(hq)), self.handle)
        out["_total_launches"] = nl.value
        out["_host_quadtree_ms"] = hq.value
        return out

    def set_camera_distortion(self, fx, fy, cx, cy, dist) -> np.ndarray:
        """Camera model of Frame::UndistortKeyPoints / ComputeImageBounds for the batched frame constructions and tracking chains of this
        context (rgbl_set_camera_distortion): K = (fx, fy, cx, cy), dist = mDistCoef (k1, k2, p1, p2[, k3]); k1 == 0 -> mvKeysUn = mvKeys.
        -> the image bounds (mnMinX, mnMaxX, mnMinY, mnMaxY)."""
        d = np.ascontiguousarray(dist, np.float32).reshape(-1)
        b = np.empty(4, np.float32)
        check(lib().rgbl_set_camera_distortion(self.handle, fx, fy, cx, cy, ptr(d), len(d), ptr(b)), self.handle)
        return b

    def set_stereo_rectification(self, m1l, m2l, m1r, m2r):
        """Rectify every later stereo pair on the device (rgbl_set_stereo_rectification): the H x W float32 maps M1l, M2l, M1r, M2r of
        cv::initUndistortRectifyMap, as Settings holds them; the stereo uploads and runners then take the raw images.  All None: off."""
        maps = [m1l, m2l, m1r, m2r]
        if all(m is None for m in maps):
            check(lib().rgbl_set_stereo_rectification(self.handle, None, None, None, None, 0), self.handle)
            return
        arr = [None if m is None else np.ascontiguousarray(m, np.float32) for m in maps]
        if any(a is not None and a.shape != (self.height, self.width) for a in arr):
            raise ValueError(f"the maps must be {self.height} x {self.width} (the context's size)")
        stride = self.width
        check(lib().rgbl_set_stereo_rectification(self.handle, *[None if a is None else ptr(a) for a in arr], stride), self.handle)

    def set_host_quadtree(self, on: bool):
        check(lib().rgbl_set_host_quadtree(self.handle, int(on)), self.handle)

    def timer_mark(self, which: int):
        check(lib().rgbl_timer_mark(self.handle, which), self.handle)

    def timer_elapsed_ms(self) -> float:
        ms = C.c_double()
        check(lib().rgbl_timer_elapsed_ms(self.handle, C.byref(ms)), self.handle)
        return ms.value

    def close(self):
        if getattr(self, "handle", None):
            lib().rgbl_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def orb_tables(nfeatures=2000, scale_factor=1.2, nlevels=8, ini_th=12, min_th=7):
    p = OrbParams(nfeatures, scale_factor, nlevels, ini_th, min_th)
    sc, inv, s2, is2 = (np.empty(nlevels, np.float32) for _ in range(4))
    q = np.empty(nlevels, np.int32); um = np.empty(16, np.int32)
    check(lib().rgbl_orb_tables(C.byref(p), ptr(sc), ptr(inv), ptr(s2), ptr(is2), ptr(q), ptr(um)))
    return dict(scale=sc, inv_scale=inv, sigma2=s2, inv_sigma2=is2, features_per_level=q, umax=um)


def decode_png_gray(ctx: "Context", png_list, camera_rgb=True):
    """cv::imread(IMREAD_UNCHANGED) + Tracking::GrabImageRGBL's cvtColor for a batch of PNG streams (rgbl_decode_png_gray)
    -> list of gray images (height x width u8)."""
    n = len(png_list)
    bufs = [np.frombuffer(b, np.uint8) for b in png_list]
    pa = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    sizes = (C.c_size_t * n)(*[len(b) for b in bufs])
    outs = [np.empty((ctx.height, ctx.width), np.uint8) for _ in range(n)]
    oa = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    check(lib().rgbl_decode_png_gray(ctx.handle, n, pa, sizes, int(bool(camera_rgb)), oa, ctx.width), ctx.handle)
    return outs


def decode_png_depth16(ctx: "Context", png_list):
    """cv::imread(IMREAD_UNCHANGED) of a batch of 16-bit depth PNG streams (rgbl_decode_png_depth16) -> list of uint16 images (H x W)."""
    n = len(png_list)
    bufs = [np.frombuffer(b, np.uint8) for b in png_list]
    pa = (C.c_void_p * n)(*[b.ctypes.data for b in bufs])
    sizes = (C.c_size_t * n)(*[len(b) for b in bufs])
    outs = [np.empty((ctx.height, ctx.width), np.uint16) for _ in range(n)]
    oa = (C.c_void_p * n)(*[o.ctypes.data for o in outs])
    check(lib().rgbl_decode_png_depth16(ctx.handle, n, pa, sizes, oa, ctx.width), ctx.handle)
    return outs


def depth_map_factor(factor: float) -> float:
    """Tracking::mDepthMapFactor from the settings' RGBD.DepthMapFactor (src/Tracking.cc:1188-1204): 1.0f / factor computed in float,
    1 when |factor| < 1e-5.  The depth_scale of the RGB-D entry points."""
    f = np.float32(factor)
    return float(np.float32(1.0) if abs(f) < np.float32(1e-5) else np.float32(1.0) / f)


class ORBextractor:
    """ORB_SLAM3::ORBextractor drop-in (src/ORBextractor.cc)."""

    def __init__(self, nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST, width, height, max_batch=1, device=0,
                 ctx: Context | None = None):
        self.ctx = ctx or Context(width, height, nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST, max_batch, 0, 0, device)
        t = orb_tables(nfeatures, scaleFactor, nlevels, iniThFAST, minThFAST)
        self.mvScaleFactor, self.mvInvScaleFactor = t["scale"], t["inv_scale"]
        self.mvLevelSigma2, self.mvInvLevelSigma2 = t["sigma2"], t["inv_sigma2"]
        self.mnFeaturesPerLevel, self.umax = t["features_per_level"], t["umax"]
        self.nlevels, self.nfeatures, self.scaleFactor = nlevels, nfeatures, scaleFactor

    # getters of include/ORBextractor.h:61-81
    def GetLevels(self): return self.nlevels
    def GetScaleFactor(self): return self.scaleFactor
    def GetScaleFactors(self): return self.mvScaleFactor
    def GetInverseScaleFactors(self): return self.mvInvScaleFactor
    def GetScaleSigmaSquares(self): return self.mvLevelSigma2
    def GetInverseScaleSigmaSquares(self): return self.mvInvLevelSigma2

    def __call__(self, image: np.ndarray, mask=None, vLappingArea=(0, 0)):
        """-> (monoIndex, keypoints[KP_DTYPE], descriptors[N,32]); monoIndex == -1 for an empty image."""
        if image is None or image.size == 0:
            return -1, np.empty(0, KP_DTYPE), np.empty((0, 32), np.uint8)
        assert image.dtype == np.uint8 and image.ndim == 2, "CV_8UC1 expected (src/ORBextractor.cc:1094)"
        img = image if image.strides[1] == 1 else np.ascontiguousarray(image)
        cap = self.ctx.cap
        kps = np.empty(cap, KP_DTYPE); desc = np.empty((cap, 32), np.uint8)
        n = C.c_int(0); mono = C.c_int(0)
        check(lib().rgbl_orb_extract(self.ctx.handle, ptr(img), img.shape[1], img.shape[0], img.strides[0],
                                     int(vLappingArea[0]), int(vLappingArea[1]), ptr(kps), ptr(desc), cap,
                                     C.byref(n), C.byref(mono)), self.ctx.handle)
        return mono.value, kps[:n.value].copy(), desc[:n.value].copy()

    def extract_batch(self, images):
        """Batched operator(): list of equally sized CV_8UC1 images -> list of (kps, desc)."""
        imgs = [np.ascontiguousarray(i, np.uint8) for i in images]
        nF = len(imgs); cap = self.ctx.cap
        arr = (C.c_void_p * nF)(*[i.ctypes.data for i in imgs])
        kps = np.empty((nF, cap), KP_DTYPE); desc = np.empty((nF, cap, 32), np.uint8)
        n = np.zeros(nF, np.int32); mono = np.zeros(nF, np.int32)
        check(lib().rgbl_orb_extract_batch(self.ctx.handle, nF, arr, imgs[0].shape[1], imgs[0].shape[0], imgs[0].strides[0],
                                           0, 0, ptr(kps), ptr(desc), cap, ptr(n), ptr(mono)), self.ctx.handle)
        return [(kps[f, :n[f]].copy(), desc[f, :n[f]].copy()) for f in range(nF)]

    # mvImagePyramid[level] (include/ORBextractor.h:83): padded plane and its ROI
    def image_pyramid_padded(self, level: int, frame: int = 0) -> np.ndarray:
        w, h = C.c_int(), C.c_int()
        buf = np.empty((self.ctx.height + 38, self.ctx.width + 38), np.uint8)
        check(lib().rgbl_orb_get_pyramid(self.ctx.handle, frame, level, ptr(buf), buf.strides[0], C.byref(w), C.byref(h)), self.ctx.handle)
        return buf[:h.value + 38, :w.value + 38].copy()

    def level_image(self, level: int, frame: int = 0) -> np.ndarray:
        w, h = C.c_int(), C.c_int()
        buf = np.empty((self.ctx.height, self.ctx.width), np.uint8)
        check(lib().rgbl_orb_get_level(self.ctx.handle, frame, level, ptr(buf), buf.strides[0], C.byref(w), C.byref(h)), self.ctx.handle)
        return buf[:h.value, :w.value].copy()

    def blurred_level(self, level: int, frame: int = 0) -> np.ndarray:
        ref = self.level_image(level, frame)
        buf = np.empty_like(ref)
        check(lib().rgbl_orb_get_blurred_level(self.ctx.handle, frame, level, ptr(buf), buf.strides[0]), self.ctx.handle)
        return buf

    def level_candidates(self, level: int, frame: int = 0) -> np.ndarray:
        cap = 1 << 18
        out = np.empty((cap, 3), np.int32); n = C.c_int(0)
        check(lib().rgbl_orb_get_candidates(self.ctx.handle, frame, level, ptr(out), cap, C.byref(n)), self.ctx.handle)
        return out[:n.value].copy()


def compute_stereo_matches(extractor: "ORBextractor", images_lr, mb: float, mbf: float):
    """Stereo Frame construction (src/Frame.cc:101-197): both images extracted as one batch, then Frame::ComputeStereoMatches.
    -> ((kps_l, desc_l), (kps_r, desc_r), mvDepth, mvuRight)"""
    (kl, dl), (kr, dr) = extractor.extract_batch(list(images_lr))
    cap = extractor.ctx.cap
    depth = np.empty(cap, np.float32); ur = np.empty(cap, np.float32)
    check(lib().rgbl_stereo_matches(extractor.ctx.handle, 0, 1, mb, mbf, ptr(depth), ptr(ur), cap), extractor.ctx.handle)
    return (kl, dl), (kr, dr), depth[:len(kl)].copy(), ur[:len(kl)].copy()


def compute_stereo_from_rgbd(ctx: Context, depth_map, kps, kps_un, bf: float):
    """Frame::ComputeStereoFromRGBD (src/Frame.cc:1074-1095): depth image H x W float32 + keypoints -> (mvDepth, mvuRight)"""
    dm = np.ascontiguousarray(depth_map, np.float32)
    kps = np.ascontiguousarray(kps, KP_DTYPE); kps_un = np.ascontiguousarray(kps_un, KP_DTYPE)
    n = len(kps)
    depth = np.empty(max(n, 1), np.float32); ur = np.empty(max(n, 1), np.float32)
    check(lib().rgbl_depth_from_map(ctx.handle, ptr(dm), dm.shape[1], dm.shape[0], dm.shape[1], bf, ptr(kps), ptr(kps_un), n, ptr(depth), ptr(ur)), ctx.handle)
    return depth[:n], ur[:n]


def stereo_matches_slots(extractor: "ORBextractor", slot_left: int, slot_right: int, n_left: int, mb: float, mbf: float):
    """Frame::ComputeStereoMatches between two frames of the last batched extraction (rgbl_stereo_matches) -> (mvDepth, mvuRight)"""
    cap = extractor.ctx.cap
    depth = np.empty(cap, np.float32); ur = np.empty(cap, np.float32)
    check(lib().rgbl_stereo_matches(extractor.ctx.handle, slot_left, slot_right, mb, mbf, ptr(depth), ptr(ur), cap), extractor.ctx.handle)
    return depth[:n_left].copy(), ur[:n_left].copy()


def fuse_search(ctx: Context, kf: FrameView, Tcw, Ow, valid, xw, normal, mf_min_dist, mf_max_dist, mp_desc, th=3.0):
    """Search part of ORBmatcher::Fuse(pKF, vpMapPoints, th) -> (bestIdx[n], bestDist[n])"""
    Tcw = np.ascontiguousarray(Tcw, np.float32); Ow = np.ascontiguousarray(Ow, np.float32); valid = np.ascontiguousarray(valid, np.uint8)
    xw = np.ascontiguousarray(xw, np.float32); normal = np.ascontiguousarray(normal, np.float32)
    mn = np.ascontiguousarray(mf_min_dist, np.float32); mx = np.ascontiguousarray(mf_max_dist, np.float32); d = np.ascontiguousarray(mp_desc, np.uint8)
    n = len(valid)
    bi = np.empty(max(n, 1), np.int32); bd = np.empty(max(n, 1), np.int32)
    nz = lambda a: ptr(a) if a.size else None
    check(lib().rgbl_fuse_search(ctx.handle, C.byref(kf.c), ptr(Tcw), ptr(Ow), n, nz(valid), nz(xw), nz(normal), nz(mn), nz(mx), nz(d), th, ptr(bi), ptr(bd)),
          ctx.handle)
    return bi[:n], bd[:n]


def distinctive_descriptors(ctx: Context, obs_start, desc):
    """MapPoint::ComputeDistinctiveDescriptors for a batch of map points (CSR of observed descriptors) -> best index per point"""
    obs_start = np.ascontiguousarray(obs_start, np.int32); desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
    best = np.empty(max(len(obs_start) - 1, 1), np.int32)
    check(lib().rgbl_distinctive_descriptors(ctx.handle, len(obs_start) - 1, ptr(obs_start), ptr(desc) if len(desc) else None, ptr(best)), ctx.handle)
    return best[:len(obs_start) - 1]


def search_for_triangulation(ctx: Context, kf1: dict, kf2: dict, F12, ep, scale_factors2, level_sigma2_2, only_stereo=False, coarse=False,
                             check_orientation=True):
    """ORBmatcher::SearchForTriangulation; kf = dict(desc, keys, has_mp, uright, fv=(node_ids, node_start, node_feat)) -> (nmatches, match12)"""
    def unpack(k):
        return (np.ascontiguousarray(k["desc"], np.uint8), np.ascontiguousarray(k["keys"]), np.ascontiguousarray(k["has_mp"], np.uint8),
                np.ascontiguousarray(k["uright"], np.float32), np.ascontiguousarray(k["fv"][0], np.uint32), np.ascontiguousarray(k["fv"][1], np.int32),
                np.ascontiguousarray(k["fv"][2], np.int32))
    d1, k1, m1, u1, i1, s1, f1 = unpack(kf1); d2, k2, m2, u2, i2, s2, f2 = unpack(kf2)
    F12 = np.ascontiguousarray(F12, np.float32).reshape(9); ep = np.ascontiguousarray(ep, np.float32)
    sf = np.ascontiguousarray(scale_factors2, np.float32); sg = np.ascontiguousarray(level_sigma2_2, np.float32)
    match = np.empty(max(len(d1), 1), np.int32); nm = C.c_int(0)
    nz = lambda a: ptr(a) if a.size else None
    check(lib().rgbl_search_for_triangulation(ctx.handle, len(d1), nz(d1), nz(k1), nz(m1), nz(u1), len(i1), nz(i1), nz(s1), nz(f1),
                                              len(d2), nz(d2), nz(k2), nz(m2), nz(u2), len(i2), nz(i2), nz(s2), nz(f2), ptr(F12), ptr(ep), len(sf), ptr(sf),
                                              ptr(sg), int(only_stereo), int(coarse), int(check_orientation), ptr(match), C.byref(nm)), ctx.handle)
    return nm.value, match[:len(d1)]


def local_bundle_adjustment(ctx: Context, poses, pose_fixed, points, e_point, e_pose, obs, stereo, inv_sigma2, fx, fy, cx, cy, bf, iterations=10):
    """Optimizer::LocalBundleAdjustment's numerical core on a flat graph (rgbl_local_bundle_adjustment)
    -> (poses[n,7], points[m,3], erase[n_edges], iterations_run)"""
    poses = np.ascontiguousarray(poses, np.float32).reshape(-1, 7); pose_fixed = np.ascontiguousarray(pose_fixed, np.uint8)
    points = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    e_point = np.ascontiguousarray(e_point, np.int32); e_pose = np.ascontiguousarray(e_pose, np.int32)
    obs = np.ascontiguousarray(obs, np.float32).reshape(-1, 3); stereo = np.ascontiguousarray(stereo, np.uint8)
    inv_sigma2 = np.ascontiguousarray(inv_sigma2, np.float32)
    po = np.empty_like(poses); pt = np.empty_like(points); er = np.zeros(max(len(e_point), 1), np.uint8); it = C.c_int(0)
    nz = lambda a: ptr(a) if a.size else None
    check(lib().rgbl_local_bundle_adjustment(ctx.handle, len(poses), nz(poses), nz(pose_fixed), len(points), nz(points), len(e_point), nz(e_point), nz(e_pose),
                                             nz(obs), nz(stereo), nz(inv_sigma2), fx, fy, cx, cy, bf, iterations, nz(po), nz(pt), ptr(er), C.byref(it)), ctx.handle)
    return po, pt, er[:len(e_point)], it.value


class ORBVocabulary:
    """DBoW2 vocabulary (ORBVocabulary = TemplatedVocabulary<FORB::TDescriptor, FORB>, include/ORBVocabulary.h) uploaded once as a
    flat tree; `transform` = Frame::ComputeBoW's mpORBvocabulary->transform(vCurrentDesc, mBowVec, mFeatVec, 4)."""

    TF_IDF, TF = 0, 1
    L1_NORM = 0

    def __init__(self, ctx: Context, child_begin, child_index, node_desc, node_weight, word_id, levels: int, weighting=0, scoring=0):
        self.ctx = ctx
        cb = np.ascontiguousarray(child_begin, np.int32); ci = np.ascontiguousarray(child_index, np.int32)
        nd = np.ascontiguousarray(node_desc, np.uint8); nw = np.ascontiguousarray(node_weight, np.float64)
        wi = np.ascontiguousarray(word_id, np.int32)
        h = C.c_void_p()
        check(lib().rgbl_vocabulary_create(ctx.handle, len(wi), ptr(cb), ptr(ci) if len(ci) else None, ptr(nd), ptr(nw), ptr(wi), int(levels),
                                           int(weighting), int(scoring), C.byref(h)), ctx.handle)
        self.handle = h

    def close(self):
        if self.handle:
            lib().rgbl_vocabulary_destroy(self.handle)
            self.handle = None

    def _out(self, n):
        return (np.empty(max(n, 1), np.int32), np.empty(max(n, 1), np.float64), np.empty(max(n, 1), np.int32), np.empty(n + 1, np.int32),
                np.empty(max(n, 1), np.int32))

    @staticmethod
    def _pack(bw, bv, nw, fn, fs, ff, nn):
        nw, nn = nw.value, nn.value
        return (bw[:nw].copy(), bv[:nw].copy()), (fn[:nn].copy(), fs[:nn + 1].copy(), ff[:fs[nn]].copy())

    def transform(self, desc, levelsup: int = 4):
        """-> (BowVector as (word ids ascending, values), FeatureVector as CSR (node ids ascending, node_start, features))"""
        desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        bw, bv, fn, fs, ff = self._out(len(desc)); nw, nn = C.c_int(0), C.c_int(0)
        check(lib().rgbl_compute_bow(self.ctx.handle, self.handle, len(desc), ptr(desc) if len(desc) else None, levelsup, ptr(bw), ptr(bv),
                                     C.byref(nw), ptr(fn), ptr(fs), ptr(ff), C.byref(nn)), self.ctx.handle)
        return self._pack(bw, bv, nw, fn, fs, ff, nn)

    def transform_resident(self, frame: int, levelsup: int = 4):
        """Same on the descriptors of frame `frame` of the context's last batched call (no upload)."""
        bw, bv, fn, fs, ff = self._out(self.ctx.cap); nw, nn = C.c_int(0), C.c_int(0)
        check(lib().rgbl_resident_compute_bow(self.ctx.handle, self.handle, frame, levelsup, ptr(bw), ptr(bv), C.byref(nw), ptr(fn), ptr(fs),
                                              ptr(ff), C.byref(nn)), self.ctx.handle)
        return self._pack(bw, bv, nw, fn, fs, ff, nn)


def structuring_element(kind: str, ku: int, kv: int | None = None) -> np.ndarray:
    kv = ku if kv is None else kv
    m = np.zeros((kv, ku), np.uint8)
    check(lib().rgbl_depth_structuring_element(kind.encode(), ku, kv, ptr(m)))
    return m


def make_depth_params(method=L.DEPTH_INVERSE_DILATION, min_dist=5.0, max_dist=200.0, bf=100.0, kernel_type="Diamond",
                      ku=5, kv=5, scale=1.0, avg_kernel=5, nn_radius=7.0) -> DepthParams:
    p = DepthParams()
    p.method, p.min_dist, p.max_dist, p.bf, p.inv_dilation_scale = method, min_dist, max_dist, bf, scale
    p.ku, p.kv = ku, kv
    m = structuring_element(kernel_type, ku, kv)
    flat = np.zeros(81, np.uint8); flat[:ku * kv] = m.reshape(-1)
    C.memmove(p.mask, flat.ctypes.data, 81)
    p.avg_kernel, p.nn_search_radius = avg_kernel, nn_radius
    return p


class DepthModule:
    """ORB_SLAM3::DepthModule drop-in for the RGB-L hot path (src/DepthModule.cc:50-274).

    The YAML parsing of the reference constructor (src/DepthModule.cc:281-601) stays with the caller;
    the parsed values are passed here (LidarProjectionMatrix, LiDAR.Method, min/max dist, kernel).
    """

    def __init__(self, ctx: Context, LidarProjectionMatrix: np.ndarray, bf: float, method="InverseDilation",
                 min_dist=5.0, max_dist=200.0, kernel_type="Diamond", kernel_size_u=5, kernel_size_v=5, avg_kernel=5, nn_radius=7.0):
        methods = {"None": L.DEPTH_NONE, "NearestNeighborPixel": L.DEPTH_NEAREST_NEIGHBOR_PIXEL,
                   "AverageFiltering": L.DEPTH_AVERAGE_FILTERING, "InverseDilation": L.DEPTH_INVERSE_DILATION}
        self.ctx = ctx
        self.LidarProjectionMatrix = np.ascontiguousarray(LidarProjectionMatrix, np.float32).reshape(3, 4)
        self.params = make_depth_params(methods[method], min_dist, max_dist, bf, kernel_type, kernel_size_u, kernel_size_v, 1.0, avg_kernel, nn_radius)
        self.mvDepth = np.empty(0, np.float32); self.mvuRight = np.empty(0, np.float32)
        self.RawDepthMap = None; self.ProcessedDepthMap = None

    def CalculateDepthFromPcd(self, mvKeys, mvKeysUn, PointCloud, imwidth, imheight, want_maps=True):
        pts = np.ascontiguousarray(PointCloud, np.float32)
        assert pts.ndim == 2 and pts.shape[0] == 4, "4 x N CV_32F point cloud expected"
        k = np.ascontiguousarray(mvKeys, KP_DTYPE); ku = np.ascontiguousarray(mvKeysUn, KP_DTYPE)
        n = len(k)
        d = np.empty(n, np.float32); u = np.empty(n, np.float32)
        raw = np.empty((imheight, imwidth), np.float32) if want_maps else None
        proc = np.empty((imheight, imwidth), np.float32) if want_maps else None
        check(lib().rgbl_depth_from_pcd(self.ctx.handle, ptr(pts), pts.shape[1], ptr(self.LidarProjectionMatrix), imwidth, imheight,
                                        C.byref(self.params), ptr(k), ptr(ku), n, ptr(d), ptr(u),
                                        ptr(raw) if want_maps else None, ptr(proc) if want_maps else None), self.ctx.handle)
        self.mvDepth, self.mvuRight, self.RawDepthMap, self.ProcessedDepthMap = d, u, raw, proc


def frame_rgbl_batch(ctx: Context, images, clouds, P, depth_params: DepthParams):
    """Fused Frame construction for n RGB-L frames (src/Frame.cc:289-377): ExtractORB + CalculateDepthFromPcd."""
    nF = len(images); cap = ctx.cap
    imgs = [np.ascontiguousarray(i, np.uint8) for i in images]
    pcs = [np.ascontiguousarray(p, np.float32) for p in clouds]
    ia = (C.c_void_p * nF)(*[i.ctypes.data for i in imgs]); pa = (C.c_void_p * nF)(*[p.ctypes.data for p in pcs])
    npts = np.array([p.shape[1] for p in pcs], np.int32)
    P = np.ascontiguousarray(P, np.float32).reshape(12)
    kps = np.empty((nF, cap), KP_DTYPE); desc = np.empty((nF, cap, 32), np.uint8)
    depth = np.empty((nF, cap), np.float32); ur = np.empty((nF, cap), np.float32); n = np.zeros(nF, np.int32)
    check(lib().rgbl_frame_rgbl_batch(ctx.handle, nF, ia, imgs[0].shape[1], imgs[0].shape[0], imgs[0].strides[0], pa, ptr(npts),
                                      ptr(P), C.byref(depth_params), ptr(kps), ptr(desc), ptr(depth), ptr(ur), cap, ptr(n)), ctx.handle)
    return [(kps[f, :n[f]].copy(), desc[f, :n[f]].copy(), depth[f, :n[f]].copy(), ur[f, :n[f]].copy()) for f in range(nF)]


class FrameView:
    """The members of ORB_SLAM3::Frame the tracking matchers read (Nleft == -1 frames), see rgbl_frame_view.  bounds = (mnMinX, mnMaxX,
    mnMinY, mnMaxY) of a distorted camera (Context.set_camera_distortion); None: (0, width, 0, height)."""

    def __init__(self, keys_un, uright, desc, width, height, scale_factors, fx, fy, cx, cy, bf, bounds=None):
        self.keys_un = np.ascontiguousarray(keys_un, KP_DTYPE)
        self.uright = np.ascontiguousarray(uright, np.float32)
        self.desc = np.ascontiguousarray(desc, np.uint8)
        self.scale_factors = np.ascontiguousarray(scale_factors, np.float32)
        self.n = len(self.keys_un)
        log_sf = float(np.float32(np.log(np.float32(self.scale_factors[1])))) if len(self.scale_factors) > 1 else 1.0
        b = (0.0, float(width), 0.0, float(height)) if bounds is None else tuple(float(v) for v in bounds)
        self.c = L.FrameViewC(self.n, self.keys_un.ctypes.data, self.uright.ctypes.data, self.desc.ctypes.data,
                              *b, len(self.scale_factors), self.scale_factors.ctypes.data,
                              fx, fy, cx, cy, bf, log_sf)


class ORBmatcher:
    """ORB_SLAM3::ORBmatcher, the tracking-thread entry points (include/ORBmatcher.h:40-69)."""

    TH_HIGH, TH_LOW, HISTO_LENGTH = 100, 50, 30

    def __init__(self, ctx: Context, nnratio=0.6, checkOri=True):
        self.ctx, self.mfNNratio, self.mbCheckOrientation = ctx, nnratio, checkOri

    @staticmethod
    def DescriptorDistance(a, b) -> int:
        a = np.ascontiguousarray(a, np.uint8); b = np.ascontiguousarray(b, np.uint8)
        return lib().rgbl_descriptor_distance(ptr(a), ptr(b))

    def SearchByProjectionLastFrame(self, cur: FrameView, cur_pose, last_pose, valid, xw, mp_desc, last_octave, last_angle,
                                    obs_pos, th, bMono=False, cur_state=None):
        """SearchByProjection(CurrentFrame, LastFrame, th, bMono) -> (nmatches, match[cur.n])"""
        cur_pose = np.ascontiguousarray(cur_pose, np.float32); last_pose = np.ascontiguousarray(last_pose, np.float32)
        valid = np.ascontiguousarray(valid, np.uint8); xw = np.ascontiguousarray(xw, np.float32)
        mp_desc = np.ascontiguousarray(mp_desc, np.uint8); last_octave = np.ascontiguousarray(last_octave, np.int32)
        last_angle = np.ascontiguousarray(last_angle, np.float32); obs_pos = np.ascontiguousarray(obs_pos, np.uint8)
        cs = None if cur_state is None else np.ascontiguousarray(cur_state, np.uint8)
        match = np.empty(cur.n, np.int32); nm = C.c_int(0)
        check(lib().rgbl_search_by_projection_last(self.ctx.handle, C.byref(cur.c), ptr(cur_pose), ptr(last_pose), len(valid), ptr(valid),
                                                   ptr(xw), ptr(mp_desc), ptr(last_octave), ptr(last_angle), ptr(obs_pos), th, int(bMono),
                                                   int(self.mbCheckOrientation), None if cs is None else ptr(cs), ptr(match), C.byref(nm)),
              self.ctx.handle)
        return nm.value, match

    def SearchByProjectionLocal(self, cur: FrameView, tr: dict, mp_desc, obs_pos, th, bFarPoints=False, thFarPoints=50.0, cur_state=None):
        """SearchByProjection(F, vpMapPoints, th, bFarPoints, thFarPoints) -> (nmatches, match[cur.n]); tr = is_in_frustum output"""
        n = len(tr["in_view"])
        mp_desc = np.ascontiguousarray(mp_desc, np.uint8); obs_pos = np.ascontiguousarray(obs_pos, np.uint8)
        cs = None if cur_state is None else np.ascontiguousarray(cur_state, np.uint8)
        match = np.empty(cur.n, np.int32); nm = C.c_int(0)
        check(lib().rgbl_search_by_projection_local(self.ctx.handle, C.byref(cur.c), n, ptr(tr["in_view"]), ptr(tr["proj_x"]), ptr(tr["proj_y"]),
                                                    ptr(tr["proj_xr"]), ptr(tr["depth"]), ptr(tr["level"]), ptr(tr["view_cos"]), ptr(mp_desc),
                                                    ptr(obs_pos), th, self.mfNNratio, int(bFarPoints), thFarPoints,
                                                    None if cs is None else ptr(cs), ptr(match), C.byref(nm)), self.ctx.handle)
        return nm.value, match


    def SearchByBoW(self, kf_desc, kf_angle, kf_valid, kf_csr, f_desc, f_angle, f_csr):
        """SearchByBoW(pKF, F, vpMapPointMatches); csr = (node_ids ascending, node_start[n+1], node_feat) -> (nmatches, match[n_f])"""
        kf_desc = np.ascontiguousarray(kf_desc, np.uint8); f_desc = np.ascontiguousarray(f_desc, np.uint8)
        kf_angle = np.ascontiguousarray(kf_angle, np.float32); f_angle = np.ascontiguousarray(f_angle, np.float32)
        kf_valid = np.ascontiguousarray(kf_valid, np.uint8)
        ki, ks, kfe = (np.ascontiguousarray(kf_csr[0], np.uint32), np.ascontiguousarray(kf_csr[1], np.int32), np.ascontiguousarray(kf_csr[2], np.int32))
        fi, fs, ffe = (np.ascontiguousarray(f_csr[0], np.uint32), np.ascontiguousarray(f_csr[1], np.int32), np.ascontiguousarray(f_csr[2], np.int32))
        match = np.empty(len(f_desc), np.int32); nm = C.c_int(0)
        check(lib().rgbl_search_by_bow(self.ctx.handle, len(kf_desc), ptr(kf_desc), ptr(kf_angle), ptr(kf_valid), len(ki), ptr(ki), ptr(ks), ptr(kfe),
                                       len(f_desc), ptr(f_desc), ptr(f_angle), len(fi), ptr(fi), ptr(fs), ptr(ffe), self.mfNNratio,
                                       int(self.mbCheckOrientation), ptr(match), C.byref(nm)), self.ctx.handle)
        return nm.value, match

    def SearchByProjectionReloc(self, cur: FrameView, cur_pose, valid, xw, mp_desc, kf_angle, mf_min, mf_max, th, ORBdist, cur_occupied=None):
        """SearchByProjection(CurrentFrame, pKF, sAlreadyFound, th, ORBdist) -> (nmatches, match[cur.n])"""
        cur_pose = np.ascontiguousarray(cur_pose, np.float32); valid = np.ascontiguousarray(valid, np.uint8)
        xw = np.ascontiguousarray(xw, np.float32); mp_desc = np.ascontiguousarray(mp_desc, np.uint8)
        kf_angle = np.ascontiguousarray(kf_angle, np.float32); mn = np.ascontiguousarray(mf_min, np.float32); mx = np.ascontiguousarray(mf_max, np.float32)
        occ = None if cur_occupied is None else np.ascontiguousarray(cur_occupied, np.uint8)
        match = np.empty(cur.n, np.int32); nm = C.c_int(0)
        check(lib().rgbl_search_by_projection_reloc(self.ctx.handle, C.byref(cur.c), ptr(cur_pose), len(valid), ptr(valid), ptr(xw), ptr(mp_desc),
                                                    ptr(kf_angle), ptr(mn), ptr(mx), th, int(ORBdist), int(self.mbCheckOrientation),
                                                    None if occ is None else ptr(occ), ptr(match), C.byref(nm)), self.ctx.handle)
        return nm.value, match


def is_in_frustum(ctx: Context, cur: FrameView, Rcw, tcw, Ow, xw, normal, mf_min_dist, mf_max_dist, cos_limit=0.5) -> dict:
    """Frame::isInFrustum over a list of map points -> dict of the mTrack* fields."""
    n = len(xw)
    Rcw = np.ascontiguousarray(Rcw, np.float32).reshape(9); tcw = np.ascontiguousarray(tcw, np.float32); Ow = np.ascontiguousarray(Ow, np.float32)
    xw = np.ascontiguousarray(xw, np.float32); normal = np.ascontiguousarray(normal, np.float32)
    mn = np.ascontiguousarray(mf_min_dist, np.float32); mx = np.ascontiguousarray(mf_max_dist, np.float32)
    out = dict(in_view=np.empty(n, np.uint8), proj_x=np.empty(n, np.float32), proj_y=np.empty(n, np.float32), proj_xr=np.empty(n, np.float32),
               depth=np.empty(n, np.float32), level=np.empty(n, np.int32), view_cos=np.empty(n, np.float32))
    check(lib().rgbl_is_in_frustum(ctx.handle, C.byref(cur.c), ptr(Rcw), ptr(tcw), ptr(Ow), n, ptr(xw), ptr(normal), ptr(mn), ptr(mx), cos_limit,
                                   ptr(out["in_view"]), ptr(out["proj_x"]), ptr(out["proj_y"]), ptr(out["proj_xr"]), ptr(out["depth"]),
                                   ptr(out["level"]), ptr(out["view_cos"])), ctx.handle)
    return out


class Optimizer:
    """ORB_SLAM3::Optimizer::PoseOptimization (src/Optimizer.cc:814-1114)."""

    @staticmethod
    def PoseOptimization(ctx: Context, pose, xw, obs, inv_sigma2, stereo, fx, fy, cx, cy, bf):
        """-> (nInliers, pose_out[7], mvbOutlier[n])"""
        pose = np.ascontiguousarray(pose, np.float32); xw = np.ascontiguousarray(xw, np.float32).reshape(-1, 3)
        obs = np.ascontiguousarray(obs, np.float32).reshape(-1, 3); inv_sigma2 = np.ascontiguousarray(inv_sigma2, np.float32)
        stereo = np.ascontiguousarray(stereo, np.uint8)
        n = len(xw)
        out = np.empty(7, np.float32); outlier = np.zeros(max(n, 1), np.uint8); ni = C.c_int(0)
        check(lib().rgbl_pose_optimize(ctx.handle, ptr(pose), n, ptr(xw), ptr(obs), ptr(inv_sigma2), ptr(stereo), fx, fy, cx, cy, bf,
                                       ptr(out), ptr(outlier), C.byref(ni)), ctx.handle)
        return ni.value, out, outlier[:n]


class ChainParams(C.Structure):
    """rgbl_chain_params (include/rgbl_b200.h)."""
    _fields_ = [("pose0", C.c_float * 7), ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("bf", C.c_float),
                ("th_last", C.c_float), ("mono", C.c_int), ("continue_sequence", C.c_int), ("local_map_frames", C.c_int),
                ("th_local", C.c_float), ("nn_ratio_local", C.c_float)]


def make_chain_params(pose0, fx, fy, cx, cy, bf, th_last=15.0, mono=False, continue_sequence=False, local_map_frames=0, th_local=3.0,
                      nn_ratio_local=0.8) -> ChainParams:
    p = ChainParams()
    for i, v in enumerate(np.asarray(pose0, np.float32).reshape(7)):
        p.pose0[i] = float(v)
    p.fx, p.fy, p.cx, p.cy, p.bf = fx, fy, cx, cy, bf
    p.th_last = th_last; p.mono = int(mono); p.continue_sequence = int(continue_sequence); p.local_map_frames = int(local_map_frames)
    p.th_local = th_local; p.nn_ratio_local = nn_ratio_local
    return p


class _FrameBatch:
    """The output buffers of one batch of frame constructions, and the calls that read the batch from the device: download,
    download_keys_un and the tracking chain.  The input kinds (RgblBatch, RgbdBatch, StereoBatch) add their inputs and upload calls."""

    def __init__(self, ctx: Context, nF: int, W: int, H: int, pinned: bool):
        self.ctx, self.nF, self.cap, self.W, self.H = ctx, nF, ctx.cap, W, H
        self._alloc = alloc = _pinned_alloc if pinned else (lambda shape, dt: np.empty(shape, dt))
        self.kps = alloc((nF, self.cap), KP_DTYPE); self.desc = alloc((nF, self.cap, 32), np.uint8)
        self.depth = alloc((nF, self.cap), np.float32); self.uright = alloc((nF, self.cap), np.float32)
        self.n = np.zeros(nF, np.int32)

    def download(self):
        c = self.ctx
        check(lib().rgbl_resident_download(c.handle, ptr(self.kps), ptr(self.desc), ptr(self.depth), ptr(self.uright), self.cap, ptr(self.n)), c.handle)
        return [(self.kps[f, :self.n[f]], self.desc[f, :self.n[f]], self.depth[f, :self.n[f]], self.uright[f, :self.n[f]]) for f in range(self.nF)]

    def download_keys_un(self):
        """mvKeysUn of the frames of the last batched call (rgbl_resident_download_keys_un): list of keypoint arrays, one per frame"""
        c = self.ctx
        kun = np.empty((self.nF, self.cap), KP_DTYPE); n = np.zeros(self.nF, np.int32)
        check(lib().rgbl_resident_download_keys_un(c.handle, ptr(kun), self.cap, ptr(n)), c.handle)
        return [kun[f, :n[f]].copy() for f in range(self.nF)]

    def track_begin2(self, prm: ChainParams):
        """rgbl_resident_track_begin2: TrackWithMotionModel + (local_map_frames > 0) TrackLocalMap per frame; continue_sequence
        tracks frame 0 of this batch against the last frame of the previous chain of this context."""
        check(lib().rgbl_resident_track_begin2(self.ctx.handle, C.byref(prm)), self.ctx.handle)

    def track_end2(self):
        """-> dict(poses[nF,7], n_matches, n_inliers, n_local_matches, n_inliers_first) of the oldest queued chain"""
        nF = self.nF
        out = dict(poses=np.empty((nF, 7), np.float32), n_matches=np.zeros(nF, np.int32), n_inliers=np.zeros(nF, np.int32),
                   n_local_matches=np.zeros(nF, np.int32), n_inliers_first=np.zeros(nF, np.int32))
        check(lib().rgbl_resident_track_end2(self.ctx.handle, ptr(out["poses"]), ptr(out["n_matches"]), ptr(out["n_inliers"]),
                                             ptr(out["n_local_matches"]), ptr(out["n_inliers_first"])), self.ctx.handle)
        return out


class RgblBatch(_FrameBatch):
    """Reusable (pinned if torch+CUDA are available) host buffers for rgbl_frame_rgbl_batch / the resident API."""

    def __init__(self, ctx: Context, images, clouds, P, depth_params: DepthParams, pinned=True):
        H, W = images[0].shape
        super().__init__(ctx, len(images), W, H, pinned)
        nF, alloc = self.nF, self._alloc
        self.img = alloc((nF, H, W), np.uint8)
        maxn = max(p.shape[1] for p in clouds)
        self.pts = alloc((nF, 4 * maxn), np.float32)
        self.npts = np.array([p.shape[1] for p in clouds], np.int32)
        for f in range(nF):
            self.img[f] = images[f]
            self.pts[f, :4 * clouds[f].shape[1]] = np.ascontiguousarray(clouds[f], np.float32).reshape(-1)
        self.ia = (C.c_void_p * nF)(*[self.img[f].ctypes.data for f in range(nF)])
        self.pa = (C.c_void_p * nF)(*[self.pts[f].ctypes.data for f in range(nF)])
        self.P = np.ascontiguousarray(P, np.float32).reshape(12)
        self.prm = depth_params
        self.h2d_bytes = int(nF * W * H + 4 * 4 * int(self.npts.sum()))

    def run_e2e(self):
        """One end-to-end call with host buffers: H2D inputs + all kernels + D2H results."""
        c = self.ctx
        check(lib().rgbl_frame_rgbl_batch(c.handle, self.nF, self.ia, self.W, self.H, self.W, self.pa, ptr(self.npts), ptr(self.P),
                                          C.byref(self.prm), ptr(self.kps), ptr(self.desc), ptr(self.depth), ptr(self.uright),
                                          self.cap, ptr(self.n)), c.handle)
        return self.n

    def d2h_bytes(self) -> int:
        return int(self.n.sum()) * (28 + 32 + 4 + 4)

    def upload(self):
        c = self.ctx
        check(lib().rgbl_resident_upload(c.handle, self.nF, self.ia, self.W, self.H, self.W, self.pa, ptr(self.npts)), c.handle)

    def upload_kitti(self, xyzr_list):
        """Resident upload with raw KITTI .bin records (n x 4: x, y, z, reflectance) instead of the planar 4 x n clouds."""
        c = self.ctx
        raw = [np.ascontiguousarray(r, np.float32).reshape(-1, 4) for r in xyzr_list]
        npts = np.array([len(r) for r in raw], np.int32)
        arr = (C.c_void_p * self.nF)(*[r.ctypes.data for r in raw])
        check(lib().rgbl_resident_upload_kitti(c.handle, self.nF, self.ia, self.W, self.H, self.W, arr, ptr(npts)), c.handle)

    def upload_kitti_png(self, png_list, xyzr_list, camera_rgb=True):
        """Resident upload with the images as PNG FILE BYTES (cv::imread + cvtColor to gray on the way, rgbl_resident_upload_kitti_png)
        and the clouds as raw KITTI .bin records."""
        c = self.ctx
        raw = [np.ascontiguousarray(r, np.float32).reshape(-1, 4) for r in xyzr_list]
        npts = np.array([len(r) for r in raw], np.int32)
        arr = (C.c_void_p * self.nF)(*[r.ctypes.data for r in raw])
        bufs = [np.frombuffer(b, np.uint8) for b in png_list]
        pa = (C.c_void_p * self.nF)(*[b.ctypes.data for b in bufs])
        sizes = (C.c_size_t * self.nF)(*[len(b) for b in bufs])
        check(lib().rgbl_resident_upload_kitti_png(c.handle, self.nF, pa, sizes, int(bool(camera_rgb)), arr, ptr(npts)), c.handle)

    def process_resident(self):
        c = self.ctx
        check(lib().rgbl_resident_process(c.handle, ptr(self.P), C.byref(self.prm), ptr(self.n)), c.handle)
        return self.n

    def track(self, pose0, fx, fy, cx, cy, bf, th=15.0, mono=False):
        """Resident tracking chain (rgbl_resident_track) -> (poses[nF,7], n_matches[nF], n_inliers[nF])"""
        c = self.ctx
        pose0 = np.ascontiguousarray(pose0, np.float32)
        poses = np.empty((self.nF, 7), np.float32); nm = np.zeros(self.nF, np.int32); ni = np.zeros(self.nF, np.int32)
        check(lib().rgbl_resident_track(c.handle, ptr(pose0), fx, fy, cx, cy, bf, th, int(mono), ptr(poses), ptr(nm), ptr(ni)), c.handle)
        return poses, nm, ni

    def track_begin(self, pose0, fx, fy, cx, cy, bf, th=15.0, mono=False):
        """Enqueue the tracking chain of the batch just processed (rgbl_resident_track_begin) and return at once; the next
        batch's process_resident / run_e2e may be issued before track_end and overlaps the chain on the device."""
        c = self.ctx
        pose0 = np.ascontiguousarray(pose0, np.float32)
        check(lib().rgbl_resident_track_begin(c.handle, ptr(pose0), fx, fy, cx, cy, bf, th, int(mono)), c.handle)

    def track_end(self):
        """Wait for the chain started by track_begin -> (poses[nF,7], n_matches[nF], n_inliers[nF])"""
        c = self.ctx
        poses = np.empty((self.nF, 7), np.float32); nm = np.zeros(self.nF, np.int32); ni = np.zeros(self.nF, np.int32)
        check(lib().rgbl_resident_track_end(c.handle, ptr(poses), ptr(nm), ptr(ni)), c.handle)
        return poses, nm, ni

    def set_inputs(self, images, clouds):
        """Refill the (pinned) input buffers with another batch of the same shape."""
        assert len(images) == self.nF
        for f in range(self.nF):
            self.img[f] = images[f]
            n = clouds[f].shape[1]
            assert 4 * n <= self.pts.shape[1]
            self.pts[f, :4 * n] = np.ascontiguousarray(clouds[f], np.float32).reshape(-1)
            self.npts[f] = n
        self.h2d_bytes = int(self.nF * self.W * self.H + 4 * 4 * int(self.npts.sum()))


class RgbdBatch(_FrameBatch):
    """Host buffers of one batch of RGB-D frames (gray image + CV_16U depth image each) for the resident RGB-D API: the RGB-D Frame
    constructor (src/Frame.cc:200-237) is upload + process_resident; download / track_begin2 / track_end2 as for RgblBatch."""

    def __init__(self, ctx: Context, images, depths, pinned=True):
        H, W = images[0].shape
        super().__init__(ctx, len(images), W, H, pinned)
        nF, alloc = self.nF, self._alloc
        self.img = alloc((nF, H, W), np.uint8); self.dep = alloc((nF, H, W), np.uint16)
        self.set_inputs(images, depths)
        self.ia = (C.c_void_p * nF)(*[self.img[f].ctypes.data for f in range(nF)])
        self.da = (C.c_void_p * nF)(*[self.dep[f].ctypes.data for f in range(nF)])

    def set_inputs(self, images, depths):
        assert len(images) == self.nF and len(depths) == self.nF
        for f in range(self.nF):
            self.img[f] = images[f]
            self.dep[f] = np.asarray(depths[f], np.uint16)

    def upload(self):
        c = self.ctx
        check(lib().rgbl_resident_upload_rgbd(c.handle, self.nF, self.ia, self.W, self.H, self.W, self.da, self.W), c.handle)

    def upload_png(self, png_list, depth_png_list, camera_rgb=True):
        """Resident upload of the files' bytes: image PNGs (imread + cvtColor to gray) and 16-bit depth PNGs (imread IMREAD_UNCHANGED)."""
        c = self.ctx
        bufs = [np.frombuffer(b, np.uint8) for b in png_list]; dbufs = [np.frombuffer(b, np.uint8) for b in depth_png_list]
        pa = (C.c_void_p * self.nF)(*[b.ctypes.data for b in bufs]); da = (C.c_void_p * self.nF)(*[b.ctypes.data for b in dbufs])
        sizes = (C.c_size_t * self.nF)(*[len(b) for b in bufs]); dsizes = (C.c_size_t * self.nF)(*[len(b) for b in dbufs])
        check(lib().rgbl_resident_upload_rgbd_png(c.handle, self.nF, pa, sizes, int(bool(camera_rgb)), da, dsizes), c.handle)

    def process_resident(self, depth_scale: float, bf: float):
        """depth_scale = Tracking::mDepthMapFactor (depth_map_factor(RGBD.DepthMapFactor)), bf = Camera.bf -> keypoints per frame"""
        c = self.ctx
        check(lib().rgbl_resident_process_rgbd(c.handle, depth_scale, bf, ptr(self.n)), c.handle)
        return self.n



class StereoBatch(_FrameBatch):
    """Host buffers of one batch of rectified stereo pairs for the resident stereo API: the stereo Frame constructor (src/Frame.cc:101-197)
    is upload + process_resident (the 2n images extracted as one batch, then ComputeStereoMatches, ctx.max_batch >= 2n); download /
    download_keys_un / track_begin2 / track_end2 then see the left frames, as for RgblBatch."""

    def __init__(self, ctx: Context, lefts, rights, pinned=True):
        H, W = lefts[0].shape
        super().__init__(ctx, len(lefts), W, H, pinned)
        nF, alloc = self.nF, self._alloc
        self.left = alloc((nF, H, W), np.uint8); self.right = alloc((nF, H, W), np.uint8)
        self.set_inputs(lefts, rights)
        self.la = (C.c_void_p * nF)(*[self.left[f].ctypes.data for f in range(nF)])
        self.ra = (C.c_void_p * nF)(*[self.right[f].ctypes.data for f in range(nF)])

    def set_inputs(self, lefts, rights):
        assert len(lefts) == self.nF and len(rights) == self.nF
        for f in range(self.nF):
            self.left[f] = lefts[f]; self.right[f] = rights[f]

    def upload(self):
        c = self.ctx
        check(lib().rgbl_resident_upload_stereo(c.handle, self.nF, self.la, self.ra, self.W, self.H, self.W), c.handle)

    def upload_png(self, left_pngs, right_pngs, camera_rgb=True):
        """Resident upload of the files' bytes (KITTI image_0 / image_1 PNGs: imread + cvtColor to gray on the way)."""
        c = self.ctx
        lb = [np.frombuffer(b, np.uint8) for b in left_pngs]; rb = [np.frombuffer(b, np.uint8) for b in right_pngs]
        la = (C.c_void_p * self.nF)(*[b.ctypes.data for b in lb]); ra = (C.c_void_p * self.nF)(*[b.ctypes.data for b in rb])
        ls = (C.c_size_t * self.nF)(*[len(b) for b in lb]); rs = (C.c_size_t * self.nF)(*[len(b) for b in rb])
        check(lib().rgbl_resident_upload_stereo_png(c.handle, self.nF, la, ls, ra, rs, int(bool(camera_rgb))), c.handle)

    def process_resident(self, mb: float, mbf: float):
        """mb = mbf / fx, mbf = Camera.bf -> keypoints per left frame"""
        c = self.ctx
        check(lib().rgbl_resident_process_stereo(c.handle, mb, mbf, ptr(self.n)), c.handle)
        return self.n


class SequenceIO(C.Structure):
    """rgbl_sequence_io (include/rgbl_b200.h)."""
    _fields_ = [("n_batches", C.c_int), ("frames_per_batch", C.c_int), ("width", C.c_int), ("height", C.c_int), ("stride", C.c_int),
                ("gray", C.c_void_p), ("pts4xn", C.c_void_p), ("n_pts", C.c_void_p), ("n_slots", C.c_int), ("first_slot", C.c_int),
                ("poses", C.c_void_p), ("n_matches", C.c_void_p), ("n_inliers", C.c_void_p), ("n_local_matches", C.c_void_p),
                ("kps", C.c_void_p), ("desc", C.c_void_p), ("depth", C.c_void_p), ("uright", C.c_void_p), ("cap", C.c_int), ("n_kp", C.c_void_p)]


class SequenceRunner:
    """rgbl_track_sequence: many consecutive batches of one RGB-L sequence per native call (the loop of Examples/RGB-L/rgbl_kitti.cc).
    Holds M batches of T frames in pinned host buffers (and, after stage(), in device slots); batches are visited round-robin."""

    def __init__(self, ctx: Context, P, depth_params: DepthParams, T: int, W: int, H: int, max_points: int, n_host_batches: int, pinned=True):
        self._init(ctx, T, W, H, n_host_batches, pinned, "rgbl", (4 * max_points,), np.float32)
        self.maxn, self.pts, self.npts = max_points, self.second, np.zeros((self.M, T), np.int32)
        self.P = np.ascontiguousarray(P, np.float32).reshape(12)
        self.prm = depth_params

    @classmethod
    def rgbd(cls, ctx: Context, depth_scale: float, bf: float, T: int, W: int, H: int, n_host_batches: int, pinned=True) -> "SequenceRunner":
        """RGB-D mode (rgbl_track_sequence_rgbd, the loop of Examples/RGB-D/rgbd_kitti.cc): batches of gray images + CV_16U depth images;
        set_batch(m, images, depths).  depth_scale = Tracking::mDepthMapFactor, bf = Camera.bf."""
        self = cls.__new__(cls)
        self._init(ctx, T, W, H, n_host_batches, pinned, "rgbd", (H, W), np.uint16)
        self.dep, self.depth_scale, self.bf = self.second, float(depth_scale), float(bf)
        return self

    @classmethod
    def stereo(cls, ctx: Context, mb: float, mbf: float, T: int, W: int, H: int, n_host_batches: int, pinned=True) -> "SequenceRunner":
        """Stereo mode (rgbl_track_sequence_stereo, the loop of Examples/Stereo/stereo_kitti.cc): batches of T rectified pairs, extracted as
        batches of 2T frames (ctx.max_batch >= 2T); set_batch(m, lefts, rights).  mb = mbf / fx, mbf = Camera.bf."""
        self = cls.__new__(cls)
        self._init(ctx, T, W, H, n_host_batches, pinned, "stereo", (H, W), np.uint8)
        self.right, self.mb, self.mbf = self.second, float(mb), float(mbf)
        return self

    def _init(self, ctx, T, W, H, n_host_batches, pinned, kind, second_shape, second_dtype):
        """The images of M batches and, per frame, the kind's second input (`second`): a flat cloud, a depth image or a right image."""
        self.ctx, self.T, self.W, self.H, self.M, self.maxn, self.kind = ctx, T, W, H, n_host_batches, 0, kind
        self._alloc = _pinned_alloc if pinned else (lambda shape, dt: np.empty(shape, dt))
        self.img = self._alloc((self.M, T, H, W), np.uint8)
        self.second = self._alloc((self.M, T) + second_shape, second_dtype)
        self._out = None

    def set_batch(self, m: int, images, clouds):
        """clouds: 4 x N point clouds (RGB-L), the uint16 depth images in RGB-D mode, or the right images in stereo mode."""
        for f in range(self.T):
            self.img[m, f] = images[f]
            if self.kind != "rgbl":
                self.second[m, f] = np.asarray(clouds[f], self.second.dtype)
                continue
            n = clouds[f].shape[1]
            self.pts[m, f, :4 * n] = np.ascontiguousarray(clouds[f], np.float32).reshape(-1)
            self.npts[m, f] = n

    def _frames(self, a, batches):
        """C array of the addresses of the frames of `batches` in a (img or second)"""
        return (C.c_void_p * (len(batches) * self.T))(*[a[m, f].ctypes.data for m in batches for f in range(self.T)])

    def stage(self, slot: int, m: int):
        """Upload host batch m into device slot `slot` (rgbl_resident_stage / _stage_rgbd / _stage_stereo)."""
        h, T, W, H = self.ctx.handle, self.T, self.W, self.H
        ia, sa = self._frames(self.img, [m]), self._frames(self.second, [m])
        if self.kind == "stereo":
            check(lib().rgbl_resident_stage_stereo(h, slot, T, ia, sa, W, H, W), h)
        elif self.kind == "rgbd":
            check(lib().rgbl_resident_stage_rgbd(h, slot, T, ia, W, H, W, sa, W), h)
        else:
            check(lib().rgbl_resident_stage(h, slot, T, ia, W, H, W, sa, ptr(np.ascontiguousarray(self.npts[m]))), h)

    def _outputs(self, nb, want_frames):
        n = nb * self.T
        key = (n, want_frames)
        if self._out is None or self._out[0] != key:
            a = self._alloc
            o = dict(poses=a((n, 7), np.float32), n_matches=a((n,), np.int32), n_inliers=a((n,), np.int32), n_local_matches=a((n,), np.int32))
            if want_frames:
                cap = self.ctx.cap
                o.update(kps=a((n, cap), KP_DTYPE), desc=a((n, cap, 32), np.uint8), depth=a((n, cap), np.float32), uright=a((n, cap), np.float32),
                         n_kp=a((n,), np.int32))
            self._out = (key, o)
        return self._out[1]

    def reserve(self, n_batches: int, want_frames: bool):
        """Allocate the (pinned) output buffers of a later run() of this size now (page-locking ~100 MB takes tens of ms)."""
        self._outputs(n_batches, want_frames)

    def run(self, chain: ChainParams, n_batches: int, first: int = 0, resident_slots: int = 0, want_frames: bool = False):
        """n_batches batches starting at host batch / device slot `first` (round-robin).  resident_slots > 0: inputs come from the staged
        device slots; else from the pinned host buffers (H2D inside the call).  -> dict of per-frame outputs (views of reused buffers)."""
        T = self.T
        o = self._outputs(n_batches, want_frames)
        io = SequenceIO()
        io.n_batches, io.frames_per_batch, io.width, io.height, io.stride = n_batches, T, self.W, self.H, self.W
        sa = na = None
        if resident_slots > 0:
            io.n_slots = resident_slots; io.first_slot = first % resident_slots
        else:
            idx = [(first + b) % self.M for b in range(n_batches)]
            ga, sa = self._frames(self.img, idx), self._frames(self.second, idx)
            io.gray = C.cast(ga, C.c_void_p)
            if self.kind == "rgbl":
                na = np.ascontiguousarray(np.concatenate([self.npts[m] for m in idx]).astype(np.int32))
                io.pts4xn = C.cast(sa, C.c_void_p); io.n_pts = na.ctypes.data
        io.poses = o["poses"].ctypes.data; io.n_matches = o["n_matches"].ctypes.data; io.n_inliers = o["n_inliers"].ctypes.data
        io.n_local_matches = o["n_local_matches"].ctypes.data
        if want_frames:
            io.kps = o["kps"].ctypes.data; io.desc = o["desc"].ctypes.data; io.depth = o["depth"].ctypes.data; io.uright = o["uright"].ctypes.data
            io.cap = self.ctx.cap; io.n_kp = o["n_kp"].ctypes.data
        h = self.ctx.handle
        if self.kind == "stereo":
            check(lib().rgbl_track_sequence_stereo(h, self.mb, self.mbf, C.byref(chain), C.byref(io), sa), h)
        elif self.kind == "rgbd":
            check(lib().rgbl_track_sequence_rgbd(h, self.depth_scale, self.bf, C.byref(chain), C.byref(io), sa, self.W), h)
        else:
            check(lib().rgbl_track_sequence(h, ptr(self.P), C.byref(self.prm), C.byref(chain), C.byref(io)), h)
        return o

    def h2d_bytes_per_batch(self) -> float:
        second = 16.0 * self.npts.sum() / self.M if self.kind == "rgbl" else self.T * self.second[0, 0].nbytes
        return float(self.T * self.W * self.H + second)

    def d2h_bytes_per_batch(self, want_frames: bool) -> float:
        b = self.T * (7 * 4 + 3 * 4)
        if want_frames:
            b += self.T * (self.ctx.cap * (28 + 32 + 4 + 4) + 4)
        return float(b)


_pinned_keep = []


def _pinned_alloc(shape, dtype):
    """numpy view of page-locked memory (torch is only the allocator here)."""
    import torch
    nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
    t = torch.empty(max(nbytes, 1), dtype=torch.uint8, pin_memory=torch.cuda.is_available())
    _pinned_keep.append(t)
    return t.numpy()[:nbytes].view(dtype).reshape(shape)

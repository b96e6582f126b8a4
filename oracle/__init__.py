"""ORACLE — test infrastructure, not product code.

ctypes front end for the CPU restatement of the reference hot path (``oracle/*_oracle.cpp``).
Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this package.  The product package
``orb_slam3_rgbl_b200`` never imports it.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_LIB_PATH = _HERE / "build" / "liborb_oracle.so"

KP_DTYPE = np.dtype([("x", "<f4"), ("y", "<f4"), ("size", "<f4"), ("angle", "<f4"),
                     ("response", "<f4"), ("octave", "<i4"), ("class_id", "<i4")])
assert KP_DTYPE.itemsize == 28


def build(force: bool = False) -> Path:
    """Compile the oracle with the committed Makefile (g++ only)."""
    srcs = list(_HERE.glob("*_oracle.cpp")) + [_HERE / "orb_pattern_31.inc", _HERE / "Makefile"]
    stale = (not _LIB_PATH.exists()) or any(s.stat().st_mtime > _LIB_PATH.stat().st_mtime for s in srcs)
    if force or stale:
        subprocess.run(["make", "-C", str(_HERE)] + (["-B"] if force else []), check=True,
                       stdout=subprocess.DEVNULL)
    return _LIB_PATH


_lib = None


_lib_override = None          # set by reference_tracking(): the wrappers below then call the reference's own code


def lib() -> C.CDLL:
    global _lib
    if _lib_override is not None:
        return _lib_override
    if _lib is None:
        if not _LIB_PATH.exists() or os.environ.get("ORACLE_REBUILD"):
            build()
        else:
            try:
                build()
            except Exception:
                pass  # prebuilt .so travels to the GPU box; make may be unnecessary there
        _lib = C.CDLL(str(_LIB_PATH))
        _declare(_lib)
    return _lib


class OrbParams(C.Structure):
    _fields_ = [("nfeatures", C.c_int), ("scale_factor", C.c_float), ("nlevels", C.c_int),
                ("ini_th", C.c_int), ("min_th", C.c_int), ("lap0", C.c_int), ("lap1", C.c_int)]


def _p(a, t=None):
    return a.ctypes.data_as(C.c_void_p)


def _declare(L):
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    L.orc_resize_linear_u8.argtypes = [vp, i, i, i, vp, i, i, i]
    L.orc_gaussian_blur7_u8.argtypes = [vp, i, i, i, vp, i]
    L.orc_fast_window.argtypes = [vp, i, i, i, i, vp, i]
    L.orc_fast_window.restype = i
    L.orc_fast_atan2.argtypes = [f, f]
    L.orc_fast_atan2.restype = f
    L.orc_distribute_quadtree.argtypes = [vp, i, i, i, i, i, i, vp, i]
    L.orc_distribute_quadtree.restype = i
    L.orc_extractor_create.argtypes = [C.POINTER(OrbParams)]
    L.orc_extractor_create.restype = vp
    L.orc_extractor_destroy.argtypes = [vp]
    L.orc_extractor_tables.argtypes = [vp, vp, vp, vp, vp]
    L.orc_extract.argtypes = [vp, vp, i, i, i, i, i, vp, vp, i, C.POINTER(i)]
    L.orc_extract.restype = i
    L.orc_level_size.argtypes = [vp, i, C.POINTER(i), C.POINTER(i)]
    L.orc_level_ptr.argtypes = [vp, i]
    L.orc_level_ptr.restype = vp
    L.orc_level_candidates.argtypes = [vp, i, vp, i]
    L.orc_level_candidates.restype = i
    L.orc_level_keypoints.argtypes = [vp, i, vp, i]
    L.orc_level_keypoints.restype = i
    L.orc_descriptor.argtypes = [vp, vp, i, vp]
    L.orc_depth_project.argtypes = [vp, i, vp, i, i, f, f, vp]
    L.orc_depth_inverse_dilation.argtypes = [vp, i, i, f, f, vp, i, i, vp]
    L.orc_depth_average_filter.argtypes = [vp, i, i, i, vp]
    L.orc_depth_gather.argtypes = [vp, i, vp, vp, i, f, vp, vp]
    L.orc_depth_nearest_neighbor_pixel.argtypes = [vp, i, i, vp, vp, i, f, f, vp, vp]
    L.orc_depth_from_pcd.argtypes = [vp, i, vp, i, i, f, f, vp, i, i, f, vp, vp, i, vp, vp, vp, vp]
    for name, (args, res) in _LATE.items():
        if hasattr(L, name):
            fn = getattr(L, name)
            fn.argtypes = args
            fn.restype = res


_LATE: dict = {}

# ------------------------------------------------------------------------------------------------
# primitives
# ------------------------------------------------------------------------------------------------

def resize_linear(src: np.ndarray, dw: int, dh: int) -> np.ndarray:
    src = np.ascontiguousarray(src, np.uint8)
    dst = np.empty((dh, dw), np.uint8)
    lib().orc_resize_linear_u8(_p(src), src.shape[1], src.shape[0], src.strides[0], _p(dst), dw, dh, dw)
    return dst


def gaussian_blur7(src: np.ndarray) -> np.ndarray:
    src = np.ascontiguousarray(src, np.uint8)
    dst = np.empty_like(src)
    lib().orc_gaussian_blur7_u8(_p(src), src.shape[1], src.shape[0], src.strides[0], _p(dst), dst.strides[0])
    return dst


def fast_window(win: np.ndarray, th: int) -> np.ndarray:
    """cv::FAST(win, th, nonmax=True) -> int32 [n,3] rows (x, y, score), row-major order."""
    win = np.ascontiguousarray(win, np.uint8)
    cap = win.size
    out = np.empty((cap, 3), np.int32)
    n = lib().orc_fast_window(_p(win), win.shape[1], win.shape[0], win.strides[0], th, _p(out), cap)
    return out[:n].copy()


def fast_atan2(y: float, x: float) -> float:
    return float(lib().orc_fast_atan2(float(y), float(x)))


def distribute_quadtree(kps: np.ndarray, min_x, max_x, min_y, max_y, n_desired) -> np.ndarray:
    kps = np.ascontiguousarray(kps, KP_DTYPE)
    out = np.empty(len(kps) + 8, KP_DTYPE)
    m = lib().orc_distribute_quadtree(_p(kps), len(kps), min_x, max_x, min_y, max_y, n_desired, _p(out), len(out))
    return out[:m].copy()


class Extractor:
    """Mirror of ORB_SLAM3::ORBextractor (include/ORBextractor.h:45-108)."""

    def __init__(self, nfeatures=2000, scale_factor=1.2, nlevels=8, ini_th=12, min_th=7):
        self.params = OrbParams(nfeatures, scale_factor, nlevels, ini_th, min_th, 0, 0)
        self.h = lib().orc_extractor_create(C.byref(self.params))
        self.nlevels = nlevels
        self.nfeatures = nfeatures
        sc = np.empty(nlevels, np.float32); inv = np.empty(nlevels, np.float32)
        q = np.empty(nlevels, np.int32); um = np.empty(16, np.int32)
        lib().orc_extractor_tables(self.h, _p(sc), _p(inv), _p(q), _p(um))
        self.scale_factors, self.inv_scale_factors, self.features_per_level, self.umax = sc, inv, q, um

    def __del__(self):
        try:
            lib().orc_extractor_destroy(self.h)
        except Exception:
            pass

    def __call__(self, img: np.ndarray, lapping=(0, 0)):
        """-> (keypoints[KP_DTYPE], descriptors[N,32] u8, mono_index)"""
        img = np.ascontiguousarray(img, np.uint8)
        cap = self.nfeatures + 64
        kps = np.empty(cap, KP_DTYPE)
        desc = np.empty((cap, 32), np.uint8)
        n = C.c_int(0)
        mono = lib().orc_extract(self.h, _p(img), img.shape[1], img.shape[0], img.strides[0],
                                 int(lapping[0]), int(lapping[1]), _p(kps), _p(desc), cap, C.byref(n))
        if mono < 0:
            raise RuntimeError(f"orc_extract failed: {mono}")
        return kps[:n.value].copy(), desc[:n.value].copy(), mono

    def level_image(self, l: int) -> np.ndarray:
        w, h = C.c_int(), C.c_int()
        lib().orc_level_size(self.h, l, C.byref(w), C.byref(h))
        ptr = lib().orc_level_ptr(self.h, l)
        buf = (C.c_uint8 * (w.value * h.value)).from_address(ptr)
        return np.frombuffer(buf, np.uint8).reshape(h.value, w.value).copy()

    def level_candidates(self, l: int) -> np.ndarray:
        cap = 1 << 18
        out = np.empty((cap, 3), np.int32)
        n = lib().orc_level_candidates(self.h, l, _p(out), cap)
        return out[:n].copy()

    def level_keypoints(self, l: int) -> np.ndarray:
        out = np.empty(self.nfeatures + 64, KP_DTYPE)
        n = lib().orc_level_keypoints(self.h, l, _p(out), len(out))
        return out[:n].copy()


def descriptor(kp, blurred: np.ndarray) -> np.ndarray:
    k = np.zeros(1, KP_DTYPE); k[0] = kp
    d = np.empty(32, np.uint8)
    blurred = np.ascontiguousarray(blurred)
    lib().orc_descriptor(_p(k), _p(blurred), blurred.strides[0], _p(d))
    return d


# ------------------------------------------------------------------------------------------------
# DepthModule
# ------------------------------------------------------------------------------------------------

def depth_project(pts4xn: np.ndarray, P: np.ndarray, W: int, H: int, min_d=5.0, max_d=200.0) -> np.ndarray:
    pts = np.ascontiguousarray(pts4xn, np.float32)
    assert pts.shape[0] == 4
    P = np.ascontiguousarray(P, np.float32).reshape(12)
    raw = np.empty((H, W), np.float32)
    lib().orc_depth_project(_p(pts), pts.shape[1], _p(P), W, H, min_d, max_d, _p(raw))
    return raw


def depth_inverse_dilation(raw: np.ndarray, mask: np.ndarray, max_d=200.0, scale=1.0) -> np.ndarray:
    raw = np.ascontiguousarray(raw, np.float32)
    mask = np.ascontiguousarray(mask, np.uint8)
    out = np.empty_like(raw)
    lib().orc_depth_inverse_dilation(_p(raw), raw.shape[1], raw.shape[0], max_d, scale, _p(mask),
                                     mask.shape[1], mask.shape[0], _p(out))
    return out


def depth_average_filter(raw: np.ndarray, k: int) -> np.ndarray:
    raw = np.ascontiguousarray(raw, np.float32)
    out = np.empty_like(raw)
    lib().orc_depth_average_filter(_p(raw), raw.shape[1], raw.shape[0], k, _p(out))
    return out


def depth_nearest_neighbor_pixel(raw: np.ndarray, kps, kps_un, bf: float, R: float = 7.0):
    raw = np.ascontiguousarray(raw, np.float32)
    kps = np.ascontiguousarray(kps, KP_DTYPE); kps_un = np.ascontiguousarray(kps_un, KP_DTYPE)
    d = np.empty(len(kps), np.float32); u = np.empty(len(kps), np.float32)
    lib().orc_depth_nearest_neighbor_pixel(_p(raw), raw.shape[1], raw.shape[0], _p(kps), _p(kps_un), len(kps), bf, R, _p(d), _p(u))
    return d, u


def depth_gather(dmap: np.ndarray, kps: np.ndarray, kps_un: np.ndarray, bf: float):
    dmap = np.ascontiguousarray(dmap, np.float32)
    kps = np.ascontiguousarray(kps, KP_DTYPE); kps_un = np.ascontiguousarray(kps_un, KP_DTYPE)
    d = np.empty(len(kps), np.float32); u = np.empty(len(kps), np.float32)
    lib().orc_depth_gather(_p(dmap), dmap.shape[1], _p(kps), _p(kps_un), len(kps), bf, _p(d), _p(u))
    return d, u


def depth_from_pcd(pts4xn, P, W, H, mask, bf, kps, kps_un, min_d=5.0, max_d=200.0):
    pts = np.ascontiguousarray(pts4xn, np.float32)
    P = np.ascontiguousarray(P, np.float32).reshape(12)
    mask = np.ascontiguousarray(mask, np.uint8)
    kps = np.ascontiguousarray(kps, KP_DTYPE); kps_un = np.ascontiguousarray(kps_un, KP_DTYPE)
    n = len(kps)
    d = np.empty(n, np.float32); u = np.empty(n, np.float32)
    raw = np.empty((H, W), np.float32); proc = np.empty((H, W), np.float32)
    lib().orc_depth_from_pcd(_p(pts), pts.shape[1], _p(P), W, H, min_d, max_d, _p(mask), mask.shape[1], mask.shape[0],
                             bf, _p(kps), _p(kps_un), n, _p(d), _p(u), _p(raw), _p(proc))
    return d, u, raw, proc


# ------------------------------------------------------------------------------------------------
# ORBmatcher / Frame grid / Optimizer::PoseOptimization
# ------------------------------------------------------------------------------------------------

class FrameViewC(C.Structure):
    _fields_ = [("n", C.c_int), ("keys_un", C.c_void_p), ("uright", C.c_void_p), ("desc", C.c_void_p),
                ("min_x", C.c_float), ("max_x", C.c_float), ("min_y", C.c_float), ("max_y", C.c_float),
                ("n_levels", C.c_int), ("scale_factors", C.c_void_p),
                ("fx", C.c_float), ("fy", C.c_float), ("cx", C.c_float), ("cy", C.c_float), ("bf", C.c_float),
                ("log_scale_factor", C.c_float)]


class FrameView:
    """The members of ORB_SLAM3::Frame the tracking matchers read (Nleft == -1)."""

    def __init__(self, keys_un, uright, desc, width, height, scale_factors, fx, fy, cx, cy, bf):
        self.keys_un = np.ascontiguousarray(keys_un, KP_DTYPE)
        self.uright = np.ascontiguousarray(uright, np.float32)
        self.desc = np.ascontiguousarray(desc, np.uint8)
        self.scale_factors = np.ascontiguousarray(scale_factors, np.float32)
        self.width, self.height = width, height
        self.fx, self.fy, self.cx, self.cy, self.bf = fx, fy, cx, cy, bf
        self.log_scale_factor = float(np.float32(np.log(np.float32(self.scale_factors[1]))))   # mfLogScaleFactor = log(mfScaleFactor)
        self.c = FrameViewC(len(self.keys_un), _p(self.keys_un), _p(self.uright), _p(self.desc), 0.0, float(width), 0.0, float(height),
                            len(self.scale_factors), _p(self.scale_factors), fx, fy, cx, cy, bf, self.log_scale_factor)


_LATE_DECL_DONE = False


def _late(L):
    global _LATE_DECL_DONE
    if _LATE_DECL_DONE:
        return
    vp, i, f = C.c_void_p, C.c_int, C.c_float
    fv = C.POINTER(FrameViewC)
    L.orc_descriptor_distance.argtypes = [vp, vp]; L.orc_descriptor_distance.restype = i
    L.orc_features_in_area.argtypes = [fv, f, f, f, i, i, vp, i]; L.orc_features_in_area.restype = i
    L.orc_search_by_projection_last.argtypes = [fv, vp, vp, i, vp, vp, vp, vp, vp, vp, f, i, i, vp, vp]
    L.orc_search_by_projection_last.restype = i
    L.orc_is_in_frustum.argtypes = [fv, vp, vp, vp, i, vp, vp, vp, vp, f, vp, vp, vp, vp, vp, vp, vp]
    L.orc_search_by_projection_local.argtypes = [fv, i, vp, vp, vp, vp, vp, vp, vp, vp, vp, f, f, i, f, vp, vp]
    L.orc_search_by_projection_local.restype = i
    L.orc_search_by_bow.argtypes = [i, vp, vp, vp, i, vp, vp, vp, i, vp, vp, i, vp, vp, vp, f, i, vp]
    L.orc_search_by_bow.restype = i
    L.orc_search_by_projection_reloc.argtypes = [fv, vp, i, vp, vp, vp, vp, vp, vp, f, i, i, vp, vp]
    L.orc_search_by_projection_reloc.restype = i
    L.orc_stereo_matches.argtypes = [i, vp, vp, i, vp, vp, i, vp, vp, vp, vp, vp, vp, f, f, vp, vp]
    L.orc_pose_optimize.argtypes = [vp, i, vp, vp, vp, vp, f, f, f, f, f, vp, vp]
    L.orc_pose_optimize.restype = i
    L.orc_compute_bow.argtypes = [i, vp, vp, vp, vp, vp, i, i, vp, i, vp, vp, C.POINTER(i), vp, vp, vp, C.POINTER(i)]
    L.orc_compute_bow.restype = i
    L.orc_local_bundle_adjustment.argtypes = [i, vp, vp, i, vp, i, vp, vp, vp, vp, vp, f, f, f, f, f, i, vp, vp, vp, vp]
    L.orc_local_bundle_adjustment.restype = i
    L.orc_fuse_search.argtypes = [fv, vp, vp, i, vp, vp, vp, vp, vp, vp, f, vp, vp]
    L.orc_distinctive_descriptors.argtypes = [i, vp, vp, vp]
    L.orc_search_for_triangulation.argtypes = [i, vp, vp, vp, vp, i, vp, vp, vp, i, vp, vp, vp, vp, i, vp, vp, vp, vp, vp, vp, vp, i, i, i, vp]
    L.orc_search_for_triangulation.restype = i
    _LATE_DECL_DONE = True


def descriptor_distance(a, b) -> int:
    _late(lib())
    a = np.ascontiguousarray(a, np.uint8); b = np.ascontiguousarray(b, np.uint8)
    return lib().orc_descriptor_distance(_p(a), _p(b))


def features_in_area(fv: FrameView, x, y, r, min_level=-1, max_level=-1) -> np.ndarray:
    _late(lib())
    out = np.empty(fv.c.n + 1, np.int32)
    n = lib().orc_features_in_area(C.byref(fv.c), x, y, r, min_level, max_level, _p(out), len(out))
    return out[:n].copy()


def search_by_projection_last(cur: FrameView, cur_pose, last_pose, valid, xw, mp_desc, last_octave, last_angle, obs_pos,
                              th, mono=False, check_orientation=True, cur_state=None):
    _late(lib())
    n_last = len(valid)
    cur_pose = np.ascontiguousarray(cur_pose, np.float32); last_pose = np.ascontiguousarray(last_pose, np.float32)
    valid = np.ascontiguousarray(valid, np.uint8); xw = np.ascontiguousarray(xw, np.float32).reshape(-1, 3)
    mp_desc = np.ascontiguousarray(mp_desc, np.uint8); last_octave = np.ascontiguousarray(last_octave, np.int32)
    last_angle = np.ascontiguousarray(last_angle, np.float32); obs_pos = np.ascontiguousarray(obs_pos, np.uint8)
    cs = np.zeros(cur.c.n, np.uint8) if cur_state is None else np.ascontiguousarray(cur_state, np.uint8)
    match = np.empty(cur.c.n, np.int32)
    nm = lib().orc_search_by_projection_last(C.byref(cur.c), _p(cur_pose), _p(last_pose), n_last, _p(valid), _p(xw), _p(mp_desc),
                                             _p(last_octave), _p(last_angle), _p(obs_pos), th, int(mono), int(check_orientation),
                                             _p(cs), _p(match))
    return nm, match


def is_in_frustum(fv: FrameView, Rcw, tcw, Ow, xw, normal, mf_min_dist, mf_max_dist, cos_limit=0.5):
    _late(lib())
    n = len(xw)
    Rcw = np.ascontiguousarray(Rcw, np.float32); tcw = np.ascontiguousarray(tcw, np.float32); Ow = np.ascontiguousarray(Ow, np.float32)
    xw = np.ascontiguousarray(xw, np.float32); normal = np.ascontiguousarray(normal, np.float32)
    mn = np.ascontiguousarray(mf_min_dist, np.float32); mx = np.ascontiguousarray(mf_max_dist, np.float32)
    out = dict(in_view=np.empty(n, np.uint8), proj_x=np.empty(n, np.float32), proj_y=np.empty(n, np.float32),
               proj_xr=np.empty(n, np.float32), depth=np.empty(n, np.float32), level=np.empty(n, np.int32), view_cos=np.empty(n, np.float32))
    lib().orc_is_in_frustum(C.byref(fv.c), _p(Rcw), _p(tcw), _p(Ow), n, _p(xw), _p(normal), _p(mn), _p(mx), cos_limit,
                            _p(out["in_view"]), _p(out["proj_x"]), _p(out["proj_y"]), _p(out["proj_xr"]), _p(out["depth"]),
                            _p(out["level"]), _p(out["view_cos"]))
    return out


def search_by_projection_local(fv: FrameView, tr: dict, mp_desc, obs_pos, th, nn_ratio=0.8, far_points=False, th_far=0.0, cur_state=None):
    _late(lib())
    n = len(tr["in_view"])
    mp_desc = np.ascontiguousarray(mp_desc, np.uint8); obs_pos = np.ascontiguousarray(obs_pos, np.uint8)
    cs = np.zeros(fv.c.n, np.uint8) if cur_state is None else np.ascontiguousarray(cur_state, np.uint8)
    match = np.empty(fv.c.n, np.int32)
    nm = lib().orc_search_by_projection_local(C.byref(fv.c), n, _p(tr["in_view"]), _p(tr["proj_x"]), _p(tr["proj_y"]), _p(tr["proj_xr"]),
                                              _p(tr["depth"]), _p(tr["level"]), _p(tr["view_cos"]), _p(mp_desc), _p(obs_pos), th, nn_ratio,
                                              int(far_points), th_far, _p(cs), _p(match))
    return nm, match


def pose_optimize(pose, xw, obs, inv_sigma2, stereo, fx, fy, cx, cy, bf):
    """-> (n_inliers, pose_out[7], outlier[n])"""
    _late(lib())
    pose = np.ascontiguousarray(pose, np.float32); xw = np.ascontiguousarray(xw, np.float32).reshape(-1, 3)
    obs = np.ascontiguousarray(obs, np.float32).reshape(-1, 3); inv_sigma2 = np.ascontiguousarray(inv_sigma2, np.float32)
    stereo = np.ascontiguousarray(stereo, np.uint8)
    n = len(xw)
    out = np.empty(7, np.float32); outlier = np.zeros(n, np.uint8)
    r = lib().orc_pose_optimize(_p(pose), n, _p(xw), _p(obs), _p(inv_sigma2), _p(stereo), fx, fy, cx, cy, bf, _p(out), _p(outlier))
    return r, out, outlier


class PoseTraceC(C.Structure):
    """PoseTrace (oracle/pose_oracle.cpp)."""
    _fields_ = [("rounds", C.c_int), ("iters", C.c_int * 4), ("rejected", C.c_int), ("max_reject_run", C.c_int),
                ("term_qmax", C.c_int), ("term_rho0", C.c_int), ("term_nbad", C.c_int), ("term_iters", C.c_int),
                ("any_sincos", C.c_int), ("empty_rounds", C.c_int), ("max_accepted_trial", C.c_int),
                ("min_rho_margin", C.c_double), ("min_stop_margin", C.c_double), ("min_chi2_margin", C.c_double)]


def pose_optimize_trace(pose, xw, obs, inv_sigma2, stereo, fx, fy, cx, cy, bf):
    """pose_optimize with the same outputs plus a dict of what the call did: rounds and LM iterations per round, rejected trials and the
    longest run of them in one iteration, how often each termination ended a round (term_qmax / term_rho0 / term_nbad / term_iters),
    whether a step had theta^2 >= 0.25 (any_sincos), rounds that began with no active edge, the highest trial index of an iteration that
    was accepted (max_accepted_trial: the damping of trial w is lambda nu^w 2^(w(w-1)/2)), and the smallest relative margins of the
    accept / reject test, the stop test and the chi2 classification (inf when no such decision depended on rounding).
    -> (n_inliers, pose_out[7], outlier[n], trace)"""
    _late(lib())
    L = lib()
    if L.orc_pose_optimize_trace.argtypes is None:
        L.orc_pose_optimize_trace.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 4 + [C.c_float] * 5 + [C.c_void_p, C.c_void_p, C.POINTER(PoseTraceC)]
        L.orc_pose_optimize_trace.restype = C.c_int
    pose = np.ascontiguousarray(pose, np.float32); xw = np.ascontiguousarray(xw, np.float32).reshape(-1, 3)
    obs = np.ascontiguousarray(obs, np.float32).reshape(-1, 3); inv_sigma2 = np.ascontiguousarray(inv_sigma2, np.float32)
    stereo = np.ascontiguousarray(stereo, np.uint8)
    n = len(xw)
    out = np.empty(7, np.float32); outlier = np.zeros(n, np.uint8); tr = PoseTraceC()
    r = L.orc_pose_optimize_trace(_p(pose), n, _p(xw), _p(obs), _p(inv_sigma2), _p(stereo), fx, fy, cx, cy, bf, _p(out), _p(outlier), C.byref(tr))
    trace = {name: (list(getattr(tr, name)) if name == "iters" else getattr(tr, name)) for name, _ in PoseTraceC._fields_}
    trace["iters"] = trace["iters"][:tr.rounds]
    return r, out, outlier, trace


def _csr(node_ids, node_start, node_feat):
    return (np.ascontiguousarray(node_ids, np.uint32), np.ascontiguousarray(node_start, np.int32), np.ascontiguousarray(node_feat, np.int32))


def search_by_bow(kf_desc, kf_angle, kf_valid, kf_csr, f_desc, f_angle, f_csr, nn_ratio=0.7, check_orientation=True):
    """SearchByBoW(KF, F): csr = (node_ids ascending, node_start[n+1], node_feat). -> (nmatches, match[n_f] = KF index or -1)"""
    _late(lib())
    kf_desc = np.ascontiguousarray(kf_desc, np.uint8); f_desc = np.ascontiguousarray(f_desc, np.uint8)
    kf_angle = np.ascontiguousarray(kf_angle, np.float32); f_angle = np.ascontiguousarray(f_angle, np.float32)
    kf_valid = np.ascontiguousarray(kf_valid, np.uint8)
    ki, ks, kfeat = _csr(*kf_csr); fi, fs, ffeat = _csr(*f_csr)
    match = np.empty(len(f_desc), np.int32)
    nm = lib().orc_search_by_bow(len(kf_desc), _p(kf_desc), _p(kf_angle), _p(kf_valid), len(ki), _p(ki), _p(ks), _p(kfeat),
                                 len(f_desc), _p(f_desc), _p(f_angle), len(fi), _p(fi), _p(fs), _p(ffeat), nn_ratio, int(check_orientation), _p(match))
    return nm, match


def search_by_projection_reloc(cur: FrameView, cur_pose, valid, xw, mp_desc, kf_angle, mf_min, mf_max, th, orb_dist, check_orientation=True, cur_occupied=None):
    _late(lib())
    cur_pose = np.ascontiguousarray(cur_pose, np.float32); valid = np.ascontiguousarray(valid, np.uint8)
    xw = np.ascontiguousarray(xw, np.float32); mp_desc = np.ascontiguousarray(mp_desc, np.uint8)
    kf_angle = np.ascontiguousarray(kf_angle, np.float32); mn = np.ascontiguousarray(mf_min, np.float32); mx = np.ascontiguousarray(mf_max, np.float32)
    occ = np.zeros(cur.c.n, np.uint8) if cur_occupied is None else np.ascontiguousarray(cur_occupied, np.uint8)
    match = np.empty(cur.c.n, np.int32)
    nm = lib().orc_search_by_projection_reloc(C.byref(cur.c), _p(cur_pose), len(valid), _p(valid), _p(xw), _p(mp_desc), _p(kf_angle), _p(mn), _p(mx),
                                              th, int(orb_dist), int(check_orientation), _p(occ), _p(match))
    return nm, match


def stereo_matches(kps_l, desc_l, kps_r, desc_r, ex_l: "Extractor", ex_r: "Extractor", mb: float, mbf: float):
    """Frame::ComputeStereoMatches on the pyramids held by two oracle extractors (after they extracted left / right)."""
    _late(lib())
    kps_l = np.ascontiguousarray(kps_l, KP_DTYPE); kps_r = np.ascontiguousarray(kps_r, KP_DTYPE)
    desc_l = np.ascontiguousarray(desc_l, np.uint8); desc_r = np.ascontiguousarray(desc_r, np.uint8)
    nl = ex_l.nlevels
    ll = [ex_l.level_image(l) for l in range(nl)]; lr = [ex_r.level_image(l) for l in range(nl)]
    pl = (C.c_void_p * nl)(*[a.ctypes.data for a in ll]); pr = (C.c_void_p * nl)(*[a.ctypes.data for a in lr])
    lw = np.array([a.shape[1] for a in ll], np.int32); lh = np.array([a.shape[0] for a in ll], np.int32)
    d = np.empty(len(kps_l), np.float32); u = np.empty(len(kps_l), np.float32)
    lib().orc_stereo_matches(len(kps_l), _p(kps_l), _p(desc_l), len(kps_r), _p(kps_r), _p(desc_r), nl, _p(ex_l.scale_factors),
                             _p(ex_l.inv_scale_factors), pl, pr, _p(lw), _p(lh), mb, mbf, _p(d), _p(u))
    return d, u


def compute_bow(vocab: dict, desc, levelsup: int = 4):
    """Frame::ComputeBoW on a flattened vocabulary dict(child_begin, child_index, node_desc, node_weight, word_id, levels)
    -> ((word ids, values), (node ids, node_start, features)) exactly as std::map iteration yields them."""
    _late(lib())
    desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32); n = len(desc)
    cb = np.ascontiguousarray(vocab["child_begin"], np.int32); ci = np.ascontiguousarray(vocab["child_index"], np.int32)
    nd = np.ascontiguousarray(vocab["node_desc"], np.uint8); nw = np.ascontiguousarray(vocab["node_weight"], np.float64)
    wi = np.ascontiguousarray(vocab["word_id"], np.int32)
    bw = np.empty(max(n, 1), np.int32); bv = np.empty(max(n, 1), np.float64)
    fn = np.empty(max(n, 1), np.int32); fs = np.empty(n + 1, np.int32); ff = np.empty(max(n, 1), np.int32)
    k, m = C.c_int(0), C.c_int(0)
    lib().orc_compute_bow(len(wi), _p(cb), _p(ci), _p(nd), _p(nw), _p(wi), int(vocab["levels"]), n, _p(desc), levelsup,
                          _p(bw), _p(bv), C.byref(k), _p(fn), _p(fs), _p(ff), C.byref(m))
    return (bw[:k.value].copy(), bv[:k.value].copy()), (fn[:m.value].copy(), fs[:m.value + 1].copy(), ff[:fs[m.value]].copy())


# ---- the reference's own DBoW2 (oracle/_ref/libref_dbow2.so, compiled unmodified from /root/reference by `make -C oracle ref`) ----
_REF_DBOW2 = _HERE / "_ref" / "libref_dbow2.so"
_ref_dbow2 = None


def ref_dbow2():
    """-> ctypes handle of the reference's DBoW2 build, or None when it is neither prebuilt nor buildable (no /root/reference)."""
    global _ref_dbow2
    if _ref_dbow2 is None:
        if not _REF_DBOW2.exists() and Path("/root/reference/Thirdparty/DBoW2").exists():
            subprocess.run(["make", "-C", str(_HERE), "ref"], check=True, stdout=subprocess.DEVNULL)
        if not _REF_DBOW2.exists():
            return None
        L = C.CDLL(str(_REF_DBOW2))
        L.ref_voc_load_text.argtypes = [C.c_char_p]; L.ref_voc_load_text.restype = C.c_void_p
        L.ref_voc_free.argtypes = [C.c_void_p]
        L.ref_voc_size.argtypes = [C.c_void_p]; L.ref_voc_size.restype = C.c_int
        L.ref_voc_transform.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                        C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.ref_voc_transform.restype = C.c_int
        _ref_dbow2 = L
    return _ref_dbow2


_REF_ORBEX = _HERE / "_ref" / "libref_orbextractor.so"
_ref_orbex = None


def ref_orbextractor():
    """-> ctypes handle of the reference's own ORBextractor.cc build (oracle/ref_orbextractor_driver.cpp), or None."""
    global _ref_orbex
    if _ref_orbex is None:
        if not _REF_ORBEX.exists() and Path("/root/reference/src/ORBextractor.cc").exists():
            subprocess.run(["make", "-C", str(_HERE), "ref"], check=True, stdout=subprocess.DEVNULL)
        if not _REF_ORBEX.exists():
            return None
        L = C.CDLL(str(_REF_ORBEX))
        L.ref_orb_extract.argtypes = [C.c_int, C.c_float, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        L.ref_orb_extract.restype = C.c_int
        L.ref_orb_tables.argtypes = [C.c_int, C.c_float, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.ref_orb_tables.restype = C.c_int
        _ref_orbex = L
    return _ref_orbex


def ref_orb_extract(img, nfeatures=2000, scale_factor=1.2, nlevels=8, ini_th=12, min_th=7, lapping=(0, 0)):
    """ORBextractor::operator() of the reference itself -> (keypoints[KP_DTYPE], descriptors, mono_index)."""
    L = ref_orbextractor()
    img = np.ascontiguousarray(img, np.uint8)
    cap = nfeatures + 64
    kps = np.empty(cap, KP_DTYPE); desc = np.empty((cap, 32), np.uint8); n = C.c_int(0)
    mono = L.ref_orb_extract(nfeatures, scale_factor, nlevels, ini_th, min_th, _p(img), img.shape[1], img.shape[0], img.strides[0],
                             int(lapping[0]), int(lapping[1]), _p(kps), _p(desc), cap, C.byref(n))
    if mono < -1:
        raise RuntimeError(f"ref_orb_extract failed: {mono}")
    return kps[:n.value].copy(), desc[:n.value].copy(), mono


_REF_DEPTH = _HERE / "_ref" / "libref_depthmodule.so"
_ref_depth = None


def ref_depthmodule():
    """-> ctypes handle of the reference's own DepthModule.cc build (oracle/ref_depthmodule_driver.cpp), or None."""
    global _ref_depth
    if _ref_depth is None:
        if not _REF_DEPTH.exists() and Path("/root/reference/src/DepthModule.cc").exists():
            subprocess.run(["make", "-C", str(_HERE), "ref"], check=True, stdout=subprocess.DEVNULL)
        if not _REF_DEPTH.exists():
            return None
        L = C.CDLL(str(_REF_DEPTH))
        L.ref_depth_from_pcd.argtypes = [C.c_char_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.ref_depth_from_pcd.restype = C.c_int
        _ref_depth = L
    return _ref_depth


def ref_depth_from_pcd(settings_path, pts4xn, W, H, kps_xy, kps_un_xy):
    """DepthModule(settings).CalculateDepthFromPcd of the reference itself -> (P[3,4], raw, processed, mvDepth, mvuRight)."""
    L = ref_depthmodule()
    pts = np.ascontiguousarray(pts4xn, np.float32)
    k = np.ascontiguousarray(kps_xy, np.float32).reshape(-1, 2); ku = np.ascontiguousarray(kps_un_xy, np.float32).reshape(-1, 2)
    P = np.empty(12, np.float32); raw = np.empty((H, W), np.float32); proc = np.empty((H, W), np.float32)
    d = np.empty(len(k), np.float32); u = np.empty(len(k), np.float32)
    rc = L.ref_depth_from_pcd(str(settings_path).encode(), _p(pts), pts.shape[1], W, H, _p(k), _p(ku), len(k), _p(P), _p(raw), _p(proc), _p(d), _p(u))
    if rc != 0:
        raise RuntimeError(f"ref_depth_from_pcd failed: {rc}")
    return P.reshape(3, 4), raw, proc, d, u


def write_vocabulary_text(vocab: dict, path, k: int) -> None:
    """A flattened vocabulary (children stored in ascending node id order, ids breadth first) in the ORBvoc.txt format that
    TemplatedVocabulary::loadFromTextFile reads (TemplatedVocabulary.h:1330-1424): header `k L scoring weighting`
    (0 0 = L1_NORM, TF_IDF as in ORBvoc.txt), then one line per node 1..n-1: parent, is-leaf, 32 descriptor bytes, weight."""
    cb, ci, nd, nw = vocab["child_begin"], vocab["child_index"], vocab["node_desc"], vocab["node_weight"]
    n = len(nw)
    parent = np.zeros(n, np.int64)
    for i in range(n):
        ch = ci[cb[i]:cb[i + 1]]
        assert (np.diff(ch) > 0).all() and (ch > i).all(), "children must be in ascending id order after their parent"
        parent[ch] = i
    with open(path, "w") as f:
        f.write(f"{k} {int(vocab['levels'])} 0 0\n")
        lines = []
        for i in range(1, n):
            leaf = 1 if cb[i + 1] == cb[i] else 0
            lines.append(f"{parent[i]} {leaf} " + " ".join(str(int(b)) for b in nd[i]) + f" {float(nw[i])!r}")
        f.write("\n".join(lines))          # no trailing newline: the loader would read an empty last line as one more node


def ref_compute_bow(voc_handle, desc, levelsup: int = 4):
    """Frame::ComputeBoW through the reference's DBoW2 itself; same return layout as compute_bow."""
    L = ref_dbow2()
    desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32); n = len(desc)
    bw = np.empty(max(n, 1), np.uint32); bv = np.empty(max(n, 1), np.float64)
    fn = np.empty(max(n, 1), np.uint32); fs = np.empty(n + 2, np.int32); ff = np.empty(max(n, 1), np.int32)
    k, m = C.c_int(0), C.c_int(0)
    rc = L.ref_voc_transform(voc_handle, _p(desc), n, levelsup, len(bw), C.byref(k), _p(bw), _p(bv), len(fn), C.byref(m), _p(fn), _p(fs), _p(ff))
    assert rc == 0
    return (bw[:k.value].astype(np.int32), bv[:k.value].copy()), (fn[:m.value].astype(np.int32), fs[:m.value + 1].copy(), ff[:fs[m.value]].copy())


def local_bundle_adjustment(poses, pose_fixed, points, e_point, e_pose, obs, stereo, inv_sigma2, fx, fy, cx, cy, bf, iterations=10):
    """Numerical core of Optimizer::LocalBundleAdjustment on a flat graph -> (poses[n,7], points[m,3], erase[n_edges], iterations, chi2)"""
    _late(lib())
    poses = np.ascontiguousarray(poses, np.float32).reshape(-1, 7); pose_fixed = np.ascontiguousarray(pose_fixed, np.uint8)
    points = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    e_point = np.ascontiguousarray(e_point, np.int32); e_pose = np.ascontiguousarray(e_pose, np.int32)
    obs = np.ascontiguousarray(obs, np.float32).reshape(-1, 3); stereo = np.ascontiguousarray(stereo, np.uint8)
    inv_sigma2 = np.ascontiguousarray(inv_sigma2, np.float32)
    po = np.empty_like(poses); pt = np.empty_like(points); er = np.zeros(len(e_point), np.uint8); chi = C.c_double(0)
    it = lib().orc_local_bundle_adjustment(len(poses), _p(poses), _p(pose_fixed), len(points), _p(points), len(e_point), _p(e_point), _p(e_pose),
                                           _p(obs), _p(stereo), _p(inv_sigma2), fx, fy, cx, cy, bf, iterations, _p(po), _p(pt), _p(er), C.byref(chi))
    return po, pt, er, it, chi.value


class BATraceC(C.Structure):
    """BATrace (oracle/ba_oracle.cpp)."""
    _fields_ = [("cap_trials", C.c_int), ("cap_iters", C.c_int),
                ("trial_lambda", C.c_void_p), ("trial_rho", C.c_void_p), ("trial_accepted", C.c_void_p), ("trial_ok", C.c_void_p),
                ("iter_qmax", C.c_void_p), ("iter_bad", C.c_void_p), ("iter_margin", C.c_void_p), ("edge_margin", C.c_void_p),
                ("n_trials", C.c_int), ("n_iters", C.c_int), ("max_reject_run", C.c_int),
                ("term_qmax", C.c_int), ("term_nbad", C.c_int), ("term_rho0", C.c_int),
                ("solver_failures", C.c_int), ("ended_on_rejected_trial", C.c_int),
                ("min_rho_margin", C.c_double), ("min_stop_margin", C.c_double), ("min_huber_margin", C.c_double),
                ("min_flag_margin", C.c_double), ("min_margin", C.c_double)]


def local_bundle_adjustment_trace(poses, pose_fixed, points, e_point, e_pose, obs, stereo, inv_sigma2, fx, fy, cx, cy, bf, iterations=10):
    """local_bundle_adjustment with the same outputs plus a dict of what the call did.  Per LM trial: trial_lambda, trial_rho,
    trial_accepted, trial_ok (the factorisation succeeded).  Per iteration: iter_qmax (trials run), iter_bad (the
    (ini - current) * 1e3 < ini decision; False when the iteration ended the run before that test) and iter_margin (its relative
    margin).  Totals: max_reject_run (most consecutive rejected trials in one iteration), term_qmax / term_nbad / term_rho0 (how the
    run ended; none set = the iteration limit), solver_failures, ended_on_rejected_trial (the erase flags then use the errors of a
    state that was not kept).  Margins (relative distance of a decision from its threshold, inf when none was taken):
    min_rho_margin (the smaller of |rho| and the relative chi2 change of the trial), min_stop_margin, min_huber_margin, min_flag_margin (chi2 against 5.991 / 7.815 and depth against 0, per edge in
    edge_margin) and min_margin, the smallest of them.
    -> (poses[n,7], points[m,3], erase[n_edges], iterations, chi2, trace)"""
    L = lib()
    _late(L)
    if L.orc_local_bundle_adjustment_trace.argtypes is None:
        L.orc_local_bundle_adjustment_trace.argtypes = L.orc_local_bundle_adjustment.argtypes + [C.POINTER(BATraceC)]
        L.orc_local_bundle_adjustment_trace.restype = C.c_int
    poses = np.ascontiguousarray(poses, np.float32).reshape(-1, 7); pose_fixed = np.ascontiguousarray(pose_fixed, np.uint8)
    points = np.ascontiguousarray(points, np.float32).reshape(-1, 3)
    e_point = np.ascontiguousarray(e_point, np.int32); e_pose = np.ascontiguousarray(e_pose, np.int32)
    obs = np.ascontiguousarray(obs, np.float32).reshape(-1, 3); stereo = np.ascontiguousarray(stereo, np.uint8)
    inv_sigma2 = np.ascontiguousarray(inv_sigma2, np.float32)
    po = np.empty_like(poses); pt = np.empty_like(points); er = np.zeros(len(e_point), np.uint8); chi = C.c_double(0)
    ct, ci = 10 * iterations + 1, iterations + 1
    arr = dict(trial_lambda=np.zeros(ct), trial_rho=np.zeros(ct), trial_accepted=np.zeros(ct, np.uint8), trial_ok=np.zeros(ct, np.uint8),
               iter_qmax=np.zeros(ci, np.int32), iter_bad=np.zeros(ci, np.uint8), iter_margin=np.full(ci, np.inf),
               edge_margin=np.full(max(len(e_point), 1), np.inf))
    tr = BATraceC(ct, ci, *[a.ctypes.data for a in arr.values()])
    it = L.orc_local_bundle_adjustment_trace(len(poses), _p(poses), _p(pose_fixed), len(points), _p(points), len(e_point), _p(e_point), _p(e_pose),
                                             _p(obs), _p(stereo), _p(inv_sigma2), fx, fy, cx, cy, bf, iterations, _p(po), _p(pt), _p(er),
                                             C.byref(chi), C.byref(tr))
    trace = {name: getattr(tr, name) for name, t in BATraceC._fields_ if t is not C.c_void_p and not name.startswith("cap_")}
    for name, a in arr.items():
        n = len(e_point) if name == "edge_margin" else (tr.n_trials if name.startswith("trial_") else tr.n_iters)
        trace[name] = a[:n].astype(bool) if a.dtype == np.uint8 else a[:n]
    return po, pt, er, it, chi.value, trace


def distinctive_descriptors(obs_start, desc):
    _late(lib())
    obs_start = np.ascontiguousarray(obs_start, np.int32); desc = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
    best = np.empty(max(len(obs_start) - 1, 1), np.int32)
    lib().orc_distinctive_descriptors(len(obs_start) - 1, _p(obs_start), _p(desc), _p(best))
    return best[:len(obs_start) - 1]


def search_for_triangulation(kf1: dict, kf2: dict, F12, ep, scale_factors2, level_sigma2_2, only_stereo=False, coarse=False, check_orientation=True):
    _late(lib())
    def unpack(k):
        return (np.ascontiguousarray(k["desc"], np.uint8), np.ascontiguousarray(k["keys"]), np.ascontiguousarray(k["has_mp"], np.uint8),
                np.ascontiguousarray(k["uright"], np.float32), np.ascontiguousarray(k["fv"][0], np.uint32), np.ascontiguousarray(k["fv"][1], np.int32),
                np.ascontiguousarray(k["fv"][2], np.int32))
    d1, k1, m1, u1, i1, s1, f1 = unpack(kf1); d2, k2, m2, u2, i2, s2, f2 = unpack(kf2)
    F12 = np.ascontiguousarray(F12, np.float32).reshape(9); ep = np.ascontiguousarray(ep, np.float32)
    sf = np.ascontiguousarray(scale_factors2, np.float32); sg = np.ascontiguousarray(level_sigma2_2, np.float32)
    match = np.empty(max(len(d1), 1), np.int32)
    nm = lib().orc_search_for_triangulation(len(d1), _p(d1), _p(k1), _p(m1), _p(u1), len(i1), _p(i1), _p(s1), _p(f1), len(d2), _p(d2), _p(k2), _p(m2), _p(u2),
                                            len(i2), _p(i2), _p(s2), _p(f2), _p(F12), _p(ep), _p(sf), _p(sg), int(only_stereo), int(coarse),
                                            int(check_orientation), _p(match))
    return nm, match[:len(d1)]


def fuse_search(kf: FrameView, Tcw, Ow, valid, xw, normal, mf_min_dist, mf_max_dist, mp_desc, th=3.0):
    _late(lib())
    Tcw = np.ascontiguousarray(Tcw, np.float32); Ow = np.ascontiguousarray(Ow, np.float32); valid = np.ascontiguousarray(valid, np.uint8)
    xw = np.ascontiguousarray(xw, np.float32); normal = np.ascontiguousarray(normal, np.float32)
    mn = np.ascontiguousarray(mf_min_dist, np.float32); mx = np.ascontiguousarray(mf_max_dist, np.float32); d = np.ascontiguousarray(mp_desc, np.uint8)
    n = len(valid)
    bi = np.empty(max(n, 1), np.int32); bd = np.empty(max(n, 1), np.int32)
    lib().orc_fuse_search(C.byref(kf.c), _p(Tcw), _p(Ow), n, _p(valid), _p(xw), _p(normal), _p(mn), _p(mx), _p(d), th, _p(bi), _p(bd))
    return bi[:n], bd[:n]


# ------------------------------------------------------------------------------------------------
# The reference's own tracking code (oracle/ref_tracking_driver.cpp -> _ref/libref_tracking.so): src/ORBmatcher.cc,
# Optimizer::PoseOptimization over the reference's g2o, Frame::isInFrustum / GetFeaturesInArea / ComputeStereoMatches ...,
# behind the same argument lists as the orc_* restatements.
# ------------------------------------------------------------------------------------------------
_REF_TRACK = _HERE / "_ref" / "libref_tracking.so"
_ref_track = None
_REF_TRACK_MIRRORED = ("descriptor_distance", "features_in_area", "search_by_projection_last", "is_in_frustum", "search_by_projection_local",
                       "search_by_bow", "search_by_projection_reloc", "pose_optimize", "stereo_matches", "distinctive_descriptors",
                       "local_bundle_adjustment")


class _RefProxy:
    """Resolves orc_<name> to ref_<name> of libref_tracking.so (same C signatures)."""

    def __init__(self, L, fallback):
        self._L = L
        self._fallback = fallback

    def __getattr__(self, name):
        if not name.startswith("orc_"):
            raise AttributeError(name)
        if name[4:] in _REF_TRACK_MIRRORED:
            return getattr(self._L, "ref_" + name[4:])
        return getattr(self._fallback, name)            # helpers the reference library has no twin of (e.g. pyramid accessors)


def ref_tracking():
    """-> proxy of the reference's own matcher / pose / stereo code, or None when it is neither prebuilt nor buildable."""
    global _ref_track
    if _ref_track is None:
        if not _REF_TRACK.exists() and Path("/root/reference/src/ORBmatcher.cc").exists():
            subprocess.run(["make", "-C", str(_HERE), "-j8", "ref"], check=True, stdout=subprocess.DEVNULL)
        if not _REF_TRACK.exists():
            return None
        o = lib(); _late(o)
        L = C.CDLL(str(_REF_TRACK))
        for name in _REF_TRACK_MIRRORED:
            src, dst = getattr(o, "orc_" + name), getattr(L, "ref_" + name)
            dst.argtypes = src.argtypes; dst.restype = src.restype
        vp, i, f = C.c_void_p, C.c_int, C.c_float
        L.ref_stereo_from_rgbd.argtypes = [i, vp, vp, vp, i, i, f, vp, vp]; L.ref_stereo_from_rgbd.restype = None
        L.ref_unproject_stereo.argtypes = [vp, i, vp, vp, f, f, f, f, vp, vp]; L.ref_unproject_stereo.restype = None
        L.ref_search_for_triangulation.argtypes = [vp, vp, f, f, f, f, i, vp, vp, vp, vp, i, vp, vp, vp, i, vp, vp, vp, vp, i, vp, vp, vp,
                                                   i, vp, vp, i, i, i, vp, vp, vp]
        L.ref_search_for_triangulation.restype = i
        L.ref_fuse.argtypes = [C.POINTER(FrameViewC), vp, i, vp, vp, vp, vp, vp, vp, f, vp, vp]; L.ref_fuse.restype = i
        _ref_track = _RefProxy(L, o)
    return _ref_track


class reference_tracking:
    """with oracle.reference_tracking(): oracle.search_by_projection_last(...) etc. run the REFERENCE's code instead of the
    restatement (same Python signatures, same arrays)."""

    def __enter__(self):
        global _lib_override
        r = ref_tracking()
        if r is None:
            raise RuntimeError("oracle/_ref/libref_tracking.so is not available")
        _late(lib())
        _lib_override = r
        return r

    def __exit__(self, *exc):
        global _lib_override
        _lib_override = None
        return False


def ref_stereo_from_rgbd(kp_xy, kp_un_xy, depth_map, mbf):
    """Frame::ComputeStereoFromRGBD of the reference itself -> (mvDepth, mvuRight)."""
    L = ref_tracking()._L
    k = np.ascontiguousarray(kp_xy, np.float32).reshape(-1, 2); ku = np.ascontiguousarray(kp_un_xy, np.float32).reshape(-1, 2)
    dm = np.ascontiguousarray(depth_map, np.float32)
    d = np.empty(len(k), np.float32); u = np.empty(len(k), np.float32)
    L.ref_stereo_from_rgbd(len(k), _p(k), _p(ku), _p(dm), dm.shape[1], dm.shape[0], mbf, _p(d), _p(u))
    return d, u


def ref_unproject_stereo(pose, kp_un_xy, depth, fx, fy, cx, cy):
    """Frame::UnprojectStereo of the reference itself for every keypoint -> (x3D[n,3], ok[n])."""
    L = ref_tracking()._L
    pose = np.ascontiguousarray(pose, np.float32); ku = np.ascontiguousarray(kp_un_xy, np.float32).reshape(-1, 2)
    depth = np.ascontiguousarray(depth, np.float32)
    x = np.empty((len(ku), 3), np.float32); ok = np.empty(len(ku), np.uint8)
    L.ref_unproject_stereo(_p(pose), len(ku), _p(ku), _p(depth), fx, fy, cx, cy, _p(x), _p(ok))
    return x, ok.astype(bool)


def ref_search_for_triangulation(T1w, T2w, cam, kf1: dict, kf2: dict, scale_factors2, level_sigma2_2, only_stereo=False, coarse=False, check_orientation=True):
    """ORBmatcher::SearchForTriangulation of the reference itself for two key frames at poses T1w / T2w (qx..tz)
    -> (nmatches, match12, F12[9] row-major, epipole[2]) - F12 and the epipole as the reference derives them from the poses."""
    L = ref_tracking()._L
    def unpack(k):
        return (np.ascontiguousarray(k["desc"], np.uint8), np.ascontiguousarray(k["keys"]), np.ascontiguousarray(k["has_mp"], np.uint8),
                np.ascontiguousarray(k["uright"], np.float32), np.ascontiguousarray(k["fv"][0], np.uint32), np.ascontiguousarray(k["fv"][1], np.int32),
                np.ascontiguousarray(k["fv"][2], np.int32))
    d1, k1, m1, u1, i1, s1, f1 = unpack(kf1); d2, k2, m2, u2, i2, s2, f2 = unpack(kf2)
    T1w = np.ascontiguousarray(T1w, np.float32); T2w = np.ascontiguousarray(T2w, np.float32)
    sf = np.ascontiguousarray(scale_factors2, np.float32); sg = np.ascontiguousarray(level_sigma2_2, np.float32)
    match = np.empty(max(len(d1), 1), np.int32); F12 = np.empty(9, np.float32); ep = np.empty(2, np.float32)
    nm = L.ref_search_for_triangulation(_p(T1w), _p(T2w), cam[0], cam[1], cam[2], cam[3], len(d1), _p(d1), _p(k1), _p(m1), _p(u1), len(i1), _p(i1), _p(s1), _p(f1),
                                        len(d2), _p(d2), _p(k2), _p(m2), _p(u2), len(i2), _p(i2), _p(s2), _p(f2), len(sf), _p(sf), _p(sg),
                                        int(only_stereo), int(coarse), int(check_orientation), _p(match), _p(F12), _p(ep))
    return nm, match[:len(d1)], F12, ep


def ref_fuse(kf: FrameView, Tcw, valid, xw, normal, mf_min_dist, mf_max_dist, mp_desc, th=3.0):
    """ORBmatcher::Fuse(pKF, vpMapPoints, th) of the reference itself -> (nFused, best_idx[n] (-1 = not fused), Ow[3])."""
    L = ref_tracking()._L
    Tcw = np.ascontiguousarray(Tcw, np.float32); valid = np.ascontiguousarray(valid, np.uint8)
    xw = np.ascontiguousarray(xw, np.float32); normal = np.ascontiguousarray(normal, np.float32)
    mn = np.ascontiguousarray(mf_min_dist, np.float32); mx = np.ascontiguousarray(mf_max_dist, np.float32); d = np.ascontiguousarray(mp_desc, np.uint8)
    n = len(valid)
    bi = np.empty(max(n, 1), np.int32); Ow = np.empty(3, np.float32)
    nf = L.ref_fuse(C.byref(kf.c), _p(Tcw), n, _p(valid), _p(xw), _p(normal), _p(mn), _p(mx), _p(d), th, _p(bi), _p(Ow))
    return nf, bi[:n], Ow


def png_decode_gray(png: bytes, camera_rgb: bool = True):
    """cv::imread(IMREAD_UNCHANGED) of a PNG stream + Tracking::GrabImageRGBL's cvtColor to gray (png_oracle.cpp)
    -> (gray[h, w] u8, pixels[h, w(, c)] u8 in FILE order R, G, B[, A])."""
    buf = np.frombuffer(png, np.uint8)
    w, h, ch = C.c_int(0), C.c_int(0), C.c_int(0)
    L = lib()
    L.orc_png_decode_gray.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    rc = L.orc_png_decode_gray(_p(buf), len(buf), int(bool(camera_rgb)), C.byref(w), C.byref(h), C.byref(ch), None, 0, None, 0)
    if rc:
        raise ValueError(f"orc_png_decode_gray: {rc}")
    gray = np.empty((h.value, w.value), np.uint8)
    px = np.empty((h.value, w.value, ch.value), np.uint8)
    rc = L.orc_png_decode_gray(_p(buf), len(buf), int(bool(camera_rgb)), C.byref(w), C.byref(h), C.byref(ch), _p(gray), gray.size, _p(px), px.size)
    if rc:
        raise ValueError(f"orc_png_decode_gray: {rc}")
    return gray, (px[..., 0] if ch.value == 1 else px)

"""Seeded problems for LocalMapping::CreateNewMapPoints (rgbl_create_new_map_points) and the CPU oracle they are checked against.

A scene is a set of 3-D points seen by key frame 1 and its neighbours: poses with real baselines, noisy projections, octaves, a
stereo fraction with depths, descriptors at controlled Hamming distances from each point's own descriptor, and feature vectors
as CSR.  Forced cases bend a scene so that a given branch of the reference's loop is reached; `tags(case, result)` lists the
branches a case reaches from the oracle's trace, and REQUIRED_TAGS is what the cases must reach together.

One branch cannot be built: an exact 0 as the 4th component of the SVD null vector (GeometricTools::Triangulate's `return
false`) needs a point at infinity that the Jacobi sweeps land on to the last bit, which no constructed input reaches reliably.
The device and the oracle both test it (tri_w0 in the trace); no case asserts that it is reached.
"""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import subprocess
import tempfile
from pathlib import Path

import numpy as np

import oracle
from orb_slam3_rgbl_b200 import _lib as L

HERE = Path(__file__).resolve().parent
FX, FY, CX, CY, BF = 400.0, 400.0, 320.0, 240.0, 40.0         # mb = 0.1
W, H = 640, 480
N_LEVELS = 8
SF = (np.float32(1.2) ** np.arange(N_LEVELS)).astype(np.float32)
SG = (SF * SF).astype(np.float32)
CAM = (FX, FY, CX, CY, BF)

ROUTES = {0: "low_parallax", 1: "triangulate", 2: "stereo1", 3: "stereo2"}
RESULTS = {0: "created", 1: "low_parallax", 2: "tri_w0", 3: "no_depth", 4: "behind1", 5: "behind2", 6: "reproj1", 7: "reproj2", 8: "dist0",
           9: "far", 10: "scale", 11: "svd_fail"}
REQUIRED_TAGS = {"route:low_parallax", "created:triangulate", "created:stereo1", "created:stereo2", "route:stereo2_both_stereo",
                 "behind1", "behind2", "reproj1:mono", "reproj1:stereo", "reproj2:mono", "reproj2:stereo", "scale", "far", "no_depth",
                 "claimed_then_absent", "duplicate_idx2", "hist_changed", "n1_strided", "no_neighbours", "empty_fv"}


# ---------------------------------------------------------------------------------------------------------------------------
# oracle: tests/new_map_points_oracle.cpp, compiled into a temporary directory keyed by its source (the tree may be read-only)
_olib = None


def _oracle_lib():
    global _olib
    if _olib is None:
        src = HERE / "new_map_points_oracle.cpp"
        key = hashlib.sha1(src.read_bytes()).hexdigest()[:12]
        out = Path(tempfile.gettempdir()) / f"rgbl_nmp_oracle_{os.getuid()}_{key}" / "libnmp_oracle.so"
        if not out.exists():
            out.parent.mkdir(parents=True, exist_ok=True)
            tmp = out.with_suffix(f".{os.getpid()}.so")
            subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-shared", "-o", str(tmp), str(src)], check=True)
            os.replace(tmp, out)
        _olib = C.CDLL(str(out))
        _olib.orc_create_new_map_points.restype = C.c_int
    return _olib


def _search_fn():
    o = oracle.lib()
    oracle._late(o)
    return C.cast(o.orc_search_for_triangulation, C.c_void_p)


def oracle_create(case, cap=None):
    """-> dict like frontend.create_new_map_points, plus trace[m, 6] = (pair, idx1, idx2, route, result, stereo flags); rc != 0 on overflow"""
    from orb_slam3_rgbl_b200.frontend import KeyFrameView
    v1 = KeyFrameView(case["kf1"]); v2 = [KeyFrameView(k) for k in case["neighbours"]]
    n = len(v2); n1 = len(v1.desc)
    arr = (L.KeyFrameViewC * max(n, 1))(*[v.c for v in v2])
    F12 = np.ascontiguousarray(case["F12"], np.float32).reshape(-1); ep = np.ascontiguousarray(case["ep"], np.float32).reshape(-1)
    if F12.size == 0:
        F12 = np.zeros(9, np.float32); ep = np.zeros(2, np.float32)
    cap = n1 if cap is None else cap
    start = np.zeros(n + 1, np.int32); nm = np.zeros(max(n, 1), np.int32)
    i1 = np.empty(max(cap, 1), np.int32); i2 = np.empty(max(cap, 1), np.int32); x = np.empty((max(cap, 1), 3), np.float32)
    trace = np.empty((max(n * n1, 1), 6), np.int32); nt = C.c_int32(0)
    p = L.ptr
    rc = _oracle_lib().orc_create_new_map_points(_search_fn(), C.byref(v1.c), C.c_int(n), arr, p(F12), p(ep), C.c_float(FX), C.c_float(FY),
                                                 C.c_float(CX), C.c_float(CY), C.c_float(BF), C.c_int(N_LEVELS), p(SF), p(SG),
                                                 C.c_float(case["th_far"]), C.c_int(int(case["check_orientation"])), C.c_int(int(case["coarse"])),
                                                 p(start), p(i1), p(i2), p(x), C.c_int(cap), p(nm), p(trace), C.byref(nt))
    m = int(start[n])
    return dict(rc=rc, created_start=start, idx1=i1[:m].copy(), idx2=i2[:m].copy(), x3d=x[:m].copy(), n_matches=nm[:n].copy(),
                trace=trace[:nt.value].copy())


def run_device(ctx, case, cap=None):
    from orb_slam3_rgbl_b200 import frontend as F
    return F.create_new_map_points(ctx, case["kf1"], case["neighbours"], case["F12"], case["ep"], CAM, N_LEVELS, SF, SG, th_far=case["th_far"],
                                   check_orientation=case["check_orientation"], coarse=case["coarse"], cap=cap)


def assert_same(got, ref):
    for k in ("created_start", "idx1", "idx2", "n_matches"):
        assert np.array_equal(got[k], ref[k]), k
    assert got["x3d"].tobytes() == ref["x3d"].tobytes(), "x3d"


# ---------------------------------------------------------------------------------------------------------------------------
# geometry
def quat_to_rot(q):
    x, y, z, w = [float(v) for v in q]
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)], [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def pose_from(rotvec, centre):
    """Tcw (qx qy qz qw tx ty tz, float32, unit quaternion) of a camera at `centre` rotated by `rotvec` (camera-to-world)"""
    th = float(np.linalg.norm(rotvec))
    ax = np.asarray(rotvec, float) / th if th > 0 else np.array([1.0, 0, 0])
    qwc = np.r_[ax * np.sin(th / 2), np.cos(th / 2)]
    qcw = np.r_[-qwc[:3], qwc[3]]
    qcw = (qcw / np.linalg.norm(qcw)).astype(np.float32)
    Rcw = quat_to_rot(qcw)
    t = -Rcw @ np.asarray(centre, float)
    return np.r_[qcw, t].astype(np.float32)


def pair_constants(T1, T2):
    """F12 = K^-T [t12]x R12 K^-1 and the epipole of camera 1 in image 2 (float64, as the shim computes them with the reference's code)"""
    R1, R2 = quat_to_rot(T1[:4]), quat_to_rot(T2[:4])
    t1, t2 = T1[4:].astype(float), T2[4:].astype(float)
    R12 = R1 @ R2.T; t12 = t1 - R12 @ t2
    K = np.array([[FX, 0, CX], [0, FY, CY], [0, 0, 1]])
    tx = np.array([[0, -t12[2], t12[1]], [t12[2], 0, -t12[0]], [-t12[1], t12[0], 0]])
    F12 = np.linalg.inv(K).T @ tx @ R12 @ np.linalg.inv(K)
    C2 = R2 @ (-R1.T @ t1) + t2
    with np.errstate(all="ignore"):
        ep = np.array([FX * C2[0] / C2[2] + CX, FY * C2[1] / C2[2] + CY])
    return F12.astype(np.float32), ep.astype(np.float32)


def _flip(rng, d, k):
    d = d.copy()
    bits = rng.choice(256, k, replace=False)
    for b in bits:
        d[b >> 3] ^= np.uint8(1 << (b & 7))
    return d


def _csr(nodes):
    order = np.argsort(nodes, kind="stable")
    ids, counts = np.unique(nodes[order], return_counts=True)
    return ids.astype(np.uint32), np.r_[0, np.cumsum(counts)].astype(np.int32), order.astype(np.int32)


class Scene:
    """n_points 3-D points in front of key frame 1 (at the origin looking down +z) and n_nb neighbours at baselines of 0.3..1.2."""

    def __init__(self, seed, n_points=300, n_nb=3, stereo=0.4, noise=0.6, n_nodes=40, extra=0.15, dist_max=12):
        self.rng = rng = np.random.default_rng(seed)
        self.P = np.c_[rng.uniform(-4, 4, n_points), rng.uniform(-3, 3, n_points), rng.uniform(3, 20, n_points)]
        self.base = rng.integers(0, 256, (n_points, 32), dtype=np.uint8)
        self.node = rng.integers(0, n_nodes, n_points)
        self.poses = [pose_from(rng.normal(0, 0.02, 3), [0, 0, 0])]
        for j in range(n_nb):
            c = rng.normal(0, 1, 3); c[2] *= 0.3
            c *= rng.uniform(0.3, 1.2) / np.linalg.norm(c)
            self.poses.append(pose_from(rng.normal(0, 0.05, 3), c))
        self.stereo, self.noise, self.extra, self.dist_max = stereo, noise, extra, dist_max

    def frame(self, k, points=None):
        """key frame k's features: one per visible point (in a shuffled order) plus unrelated features"""
        rng = self.rng
        T = self.poses[k]; R = quat_to_rot(T[:4]); t = T[4:].astype(float)
        pts = np.arange(len(self.P)) if points is None else np.asarray(points)
        Pc = self.P[pts] @ R.T + t
        u = FX * Pc[:, 0] / Pc[:, 2] + CX; v = FY * Pc[:, 1] / Pc[:, 2] + CY
        vis = (Pc[:, 2] > 0.5) & (u > 0) & (u < W) & (v > 0) & (v < H)
        pts, Pc, u, v = pts[vis], Pc[vis], u[vis], v[vis]
        n_extra = int(self.extra * len(pts))
        n = len(pts) + n_extra
        keys_un = np.zeros(n, L.KP_DTYPE)
        oct_ = rng.integers(0, 4, n)
        s = SF[oct_]
        keys_un["x"][:len(pts)] = u + rng.normal(0, self.noise, len(pts)) * s[:len(pts)]
        keys_un["y"][:len(pts)] = v + rng.normal(0, self.noise, len(pts)) * s[:len(pts)]
        keys_un["x"][len(pts):] = rng.uniform(0, W, n_extra); keys_un["y"][len(pts):] = rng.uniform(0, H, n_extra)
        keys_un["octave"] = oct_; keys_un["size"] = 31 * s; keys_un["angle"] = rng.uniform(0, 1, n)
        keys = keys_un.copy(); keys["x"] += 0.7; keys["y"] -= 0.4            # mvKeys: the distorted positions differ
        desc = np.empty((n, 32), np.uint8)
        for i, p in enumerate(pts):
            desc[i] = _flip(rng, self.base[p], int(rng.integers(0, self.dist_max)))
        desc[len(pts):] = rng.integers(0, 256, (n_extra, 32), dtype=np.uint8)
        z = np.r_[Pc[:, 2], rng.uniform(3, 20, n_extra)]
        st = rng.random(n) < self.stereo
        depth = np.where(st, z * (1 + rng.normal(0, 0.002, n)), -1).astype(np.float32)
        uright = np.where(st, keys_un["x"] - BF / np.maximum(depth, 1e-3), -1).astype(np.float32)
        nodes = np.r_[self.node[pts], rng.integers(0, self.node.max() + 1, n_extra)]
        perm = rng.permutation(n)
        inv = np.argsort(perm)
        f = dict(desc=desc[perm], keys=keys[perm], keys_un=keys_un[perm], uright=uright[perm], depth=depth[perm],
                 has_mp=(rng.random(n) < 0.1)[perm].astype(np.uint8), Tcw=T, point=np.r_[pts, -np.ones(n_extra, int)][perm])
        f["fv"] = _csr(nodes[perm])
        f["_inv"] = inv
        return f

    def case(self, name, nb=None, th_far=0.0, check_orientation=False, coarse=False, **kw):
        kf1 = self.frame(0)
        nbs = [self.frame(k) for k in (range(1, len(self.poses)) if nb is None else nb)]
        return make_case(name, kf1, nbs, th_far=th_far, check_orientation=check_orientation, coarse=coarse, **kw)


def make_case(name, kf1, nbs, th_far=0.0, check_orientation=False, coarse=False, expect=()):
    F12 = np.zeros((len(nbs), 9), np.float32); ep = np.zeros((len(nbs), 2), np.float32)
    for j, k in enumerate(nbs):
        f, e = pair_constants(kf1["Tcw"], k["Tcw"])
        F12[j] = f.reshape(9); ep[j] = e
    return dict(name=name, kf1=kf1, neighbours=nbs, F12=F12, ep=ep, th_far=th_far, check_orientation=check_orientation, coarse=coarse,
                expect=set(expect))


def feature_of(f, point):
    idx = np.nonzero(f["point"] == point)[0]
    return int(idx[0]) if len(idx) else -1


# ---------------------------------------------------------------------------------------------------------------------------
# forced cases
def case_branches(seed=11):
    """a mixed scene, then individual features bent towards each reject branch of the loop body"""
    s = Scene(seed, n_points=260, n_nb=2, stereo=0.5)
    c = s.case("branches", expect={"reproj1:stereo", "scale", "no_depth", "created:triangulate", "claimed_then_absent"})
    kf1, nb = c["kf1"], c["neighbours"][0]
    rng = np.random.default_rng(seed)
    found = {"mono": 0, "stereo": 0}
    for p in rng.permutation(len(s.P)):
        i1, i2 = feature_of(kf1, p), feature_of(nb, p)
        if i1 < 0 or i2 < 0:
            continue
        kf1["has_mp"][i1] = 0; nb["has_mp"][i2] = 0
        kind = "stereo" if kf1["uright"][i1] >= 0 else "mono"
        if found[kind] < 3:                          # a reprojection outlier in key frame 1 (several: some are rejected earlier)
            kf1["keys_un"]["y"][i1] += 9.0 * SF[kf1["keys_un"]["octave"][i1]]
        elif found[kind] < 6:                        # ... and in key frame 2
            nb["keys_un"]["y"][i2] += 9.0 * SF[nb["keys_un"]["octave"][i2]]
        elif found[kind] < 8:                        # scale inconsistency: octaves far apart
            kf1["keys_un"]["octave"][i1] = 0; nb["keys_un"]["octave"][i2] = 7
        elif found[kind] < 9 and kind == "stereo":   # stereo without depth
            kf1["depth"][i1] = 0.0
        found[kind] += 1
    # behind the cameras: stereo depth that puts the point behind camera 2 / a far-off mismatch whose rays cross behind camera 1
    for k, p in enumerate(rng.permutation(len(s.P))[:40]):
        i1, i2 = feature_of(kf1, p), feature_of(nb, p)
        if i1 < 0 or i2 < 0:
            continue
        kf1["has_mp"][i1] = 0; nb["has_mp"][i2] = 0
        nb["uright"][i2] = -1; nb["depth"][i2] = -1
        if k % 2 == 0:
            kf1["uright"][i1] = kf1["keys_un"]["x"][i1] - 1.0; kf1["depth"][i1] = -0.5 if k % 4 == 0 else 60.0
        else:
            kf1["uright"][i1] = -1; kf1["depth"][i1] = -1
            nb["keys_un"]["x"][i2] = 2 * CX - nb["keys_un"]["x"][i2]
    return c


def manual_case(name, centres, items, check_orientation=False, expect=(), seed=0):
    """key frame 1 at the origin and unrotated neighbours at `centres`; each item is one match of neighbour item["nb"]: the projections
    of the world point Q into both cameras (a point behind a camera projects to the mirrored pixel, which a ray through it reaches),
    stereo depths st1 / st2 (None: mono; uright consistent with the given depth), octaves, angles.  Items with the same "key" share
    their key-frame-1 feature.  Descriptors are random per feature and equal between the two sides of a match; one vocabulary node."""
    rng = np.random.default_rng(seed)
    proj = lambda Q, c: (FX * (Q[0] - c[0]) / (Q[2] - c[2]) + CX, FY * (Q[1] - c[1]) / (Q[2] - c[2]) + CY)
    f1, f2 = [], [[] for _ in centres]
    keyed = {}
    for it in items:
        Q = np.asarray(it["Q"], float)
        if it.get("key") in keyed:
            i1 = keyed[it["key"]]
        else:
            i1 = len(f1)
            f1.append(dict(uv=proj(Q, (0, 0, 0)), st=it.get("st1"), oct=it.get("oct1", 0), ang=it.get("ang1", 0.0), desc=rng.integers(0, 256, 32, dtype=np.uint8)))
            if "key" in it:
                keyed[it["key"]] = i1
        f2[it["nb"]].append(dict(uv=proj(Q, centres[it["nb"]]), st=it.get("st2"), oct=it.get("oct2", 0), ang=it.get("ang2", 0.0), desc=f1[i1]["desc"]))

    def frame(fs, T):
        n = len(fs)
        k = np.zeros(n, L.KP_DTYPE)
        k["x"] = [f["uv"][0] for f in fs]; k["y"] = [f["uv"][1] for f in fs]; k["octave"] = [f["oct"] for f in fs]; k["angle"] = [f["ang"] for f in fs]
        k["size"] = 31
        depth = np.array([f["st"] if f["st"] is not None else -1 for f in fs], np.float32)
        ur = np.where(depth > 0, k["x"] - BF / np.where(depth > 0, depth, 1), -1).astype(np.float32)
        ur[[f["st"] is not None and f["st"] <= 0 for f in fs]] = 1.0          # stereo flag without a usable depth
        desc = np.array([f["desc"] for f in fs], np.uint8).reshape(n, 32)
        fv = (np.array([7], np.uint32), np.array([0, n], np.int32), np.arange(n, dtype=np.int32)) if n else \
             (np.zeros(0, np.uint32), np.zeros(1, np.int32), np.zeros(0, np.int32))
        return dict(desc=desc, keys=k, keys_un=k.copy(), uright=ur, depth=depth, has_mp=np.zeros(n, np.uint8), Tcw=T, fv=fv, point=np.arange(n))
    kf1 = frame(f1, pose_from([0, 0, 0], [0, 0, 0]))
    nbs = [frame(f2[j], pose_from([0, 0, 0], c)) for j, c in enumerate(centres)]
    return make_case(name, kf1, nbs, check_orientation=check_orientation, expect=expect)


def case_forced(seed=12):
    """one match per branch that needs exact geometry: behind either camera, the stereo-2 branch with both features stereo (rays more than
    90 degrees apart, so only cosParallaxStereo1 is set by the `else if`), reprojection outliers from a wrong stereo depth"""
    C0, C1, C2 = (0.3, 0.0, 1.0), (0.3, 0.0, -1.0), (0.3, 0.0, 0.0)
    items = [dict(nb=0, Q=(0.1, 0.05, 0.6)),                                  # in front of camera 1, behind camera 2
             dict(nb=1, Q=(0.2, 0.05, -0.4)),                                 # behind camera 1, in front of camera 2
             dict(nb=0, Q=(-0.5, 0.0, 0.8), st1=3.0, st2=1.0),                # rays > 90 degrees apart, both stereo
             dict(nb=2, Q=(0.4, -0.3, 10.0), st1=1.0),                        # kf1 depth 1 instead of 10: stereo 1, kf2 mono fails
             dict(nb=2, Q=(-0.4, 0.3, 10.0), st1=1.0, st2=10.0),              # ... kf2 stereo fails
             dict(nb=2, Q=(0.6, 0.2, 10.0), st2=1.0),                         # kf2 depth 1: stereo 2, kf1 mono fails
             dict(nb=2, Q=(-0.6, -0.2, 10.0), st1=0.0, st2=0.5),              # stereo 1 without depth
             dict(nb=2, Q=(0.1, 0.1, 8.0)), dict(nb=2, Q=(-0.2, 0.4, 9.0), st1=9.0)]
    return manual_case("forced", [C0, C1, C2], items, seed=seed,
                       expect={"behind1", "behind2", "route:stereo2_both_stereo", "reproj2:mono", "reproj2:stereo", "reproj1:mono", "no_depth",
                               "created:triangulate"})


def case_low_parallax(seed=13):
    """a neighbour at the minimum baseline and far points, mostly mono: many rays closer than 0.9998"""
    s = Scene(seed, n_points=200, n_nb=1, stereo=0.1)
    s.P[:, 2] = s.P[:, 2] * 8
    s.poses[1] = pose_from([0, 0, 0], [0.1, 0, 0])
    return s.case("low_parallax", expect={"route:low_parallax"})


def case_far(seed=14):
    return Scene(seed, n_points=200, n_nb=2).case("far", th_far=11.0, expect={"far"})


def case_claimed(seed=15):
    """neighbours 0 and 1 see the same points: what neighbour 0 creates is absent from neighbour 1's search"""
    s = Scene(seed, n_points=200, n_nb=2, stereo=0.3)
    return s.case("claimed", expect={"claimed_then_absent"})


def case_duplicate(seed=16):
    """two key-frame-1 features with one descriptor and nearby keypoints match the same key-frame-2 feature"""
    s = Scene(seed, n_points=150, n_nb=1, stereo=0.0, dist_max=2)
    c = s.case("duplicate", expect={"duplicate_idx2"})
    kf1 = c["kf1"]
    cand = [i for i in range(len(kf1["desc"])) if kf1["point"][i] >= 0][:20]
    add = {k: [] for k in ("desc", "keys", "keys_un", "uright", "depth", "has_mp", "point")}
    for i in cand:
        for k in add:
            add[k].append(kf1[k][i])
    n0 = len(kf1["desc"])
    for k in add:
        kf1[k] = np.concatenate([kf1[k], np.array(add[k], dtype=kf1[k].dtype)])
    kf1["keys_un"]["x"][n0:] += 0.3
    kf1["uright"][n0:] = -1; kf1["depth"][n0:] = -1; kf1["uright"][cand] = -1; kf1["depth"][cand] = -1
    kf1["has_mp"][:] = 0; kf1["has_mp"][n0:] = 0
    nodes = np.empty(len(kf1["desc"]), np.int64)
    ids, start, feat = kf1["fv"]
    for a in range(len(ids)):
        nodes[feat[start[a]:start[a + 1]]] = ids[a]
    nodes[n0:] = nodes[cand]
    kf1["fv"] = _csr(nodes)
    c["neighbours"][0]["has_mp"][:] = 0
    return c


def case_orientation(seed=17):
    """check_orientation: neighbour 0 creates the 30 points whose rotation bin (0) dominates neighbour 1's histogram; over the surviving
    matches neighbour 1's three maxima are bins 5, 10 and 15, over all matches 0, 5 and 10: bin 15 is kept only because of the masking"""
    rng = np.random.default_rng(seed)
    items = []
    for k in range(30):
        Q = (rng.uniform(-2, 2), rng.uniform(-1.5, 1.5), rng.uniform(5, 10))
        items += [dict(nb=0, Q=Q, key=k), dict(nb=1, Q=Q, key=k)]
    for b, cnt in ((5, 5), (10, 5), (15, 4)):
        for _ in range(cnt):
            items.append(dict(nb=1, Q=(rng.uniform(-2, 2), rng.uniform(-1.5, 1.5), rng.uniform(5, 10)), ang1=30.0 * b))
    return manual_case("orientation", [(0.5, 0.0, 0.1), (-0.6, 0.1, 0.0)], items, check_orientation=True, expect={"hist_changed"}, seed=seed)


def case_large(seed=18):
    """n1 > 1024: the ordered pass's chunks and the strided histogram"""
    return Scene(seed, n_points=1400, n_nb=3, extra=0.1).case("large", check_orientation=True, expect={"n1_strided"})


def case_no_neighbours(seed=19):
    s = Scene(seed, n_points=50, n_nb=0)
    return s.case("no_neighbours", expect={"no_neighbours"})


def case_empty_fv(seed=20):
    s = Scene(seed, n_points=80, n_nb=2)
    c = s.case("empty_fv", expect={"empty_fv"})
    c["neighbours"][1]["fv"] = (np.zeros(0, np.uint32), np.zeros(1, np.int32), np.zeros(0, np.int32))
    return c


def case_coarse(seed=21):
    return Scene(seed, n_points=200, n_nb=2).case("coarse", coarse=True)


def all_cases():
    return [case_branches(), case_forced(), case_low_parallax(), case_far(), case_claimed(), case_duplicate(), case_orientation(), case_large(),
            case_no_neighbours(), case_empty_fv(), case_coarse()]


def emulated_cases():
    """a subset small enough for the CPU emulation that still reaches every tag (with the capacity check, which every case can take)"""
    names = {"branches", "forced", "low_parallax", "far", "claimed", "duplicate", "orientation", "no_neighbours", "empty_fv"}
    return [c for c in all_cases() if c["name"] in names]


def full_scene(seed):
    """key frame 1 with about 2000 features and 10 neighbours"""
    s = Scene(1000 + seed, n_points=1850, n_nb=10, stereo=0.4, n_nodes=400, extra=0.1)
    s.P[:, 0] *= 0.8
    return s.case(f"scene{seed}", check_orientation=bool(seed % 2))


# ---------------------------------------------------------------------------------------------------------------------------
def search_with_carried(case, ref):
    """(n_matches per pair, match12 per pair) from the oracle's SearchForTriangulation with has_mp1 carried as the reference does"""
    kf1 = dict(case["kf1"]); has = kf1["has_mp"].astype(np.uint8).copy()
    out = []
    for j, nb in enumerate(case["neighbours"]):
        k1 = dict(desc=kf1["desc"], keys=kf1["keys_un"], has_mp=has.copy(), uright=kf1["uright"], fv=kf1["fv"])
        k2 = dict(desc=nb["desc"], keys=nb["keys_un"], has_mp=nb["has_mp"], uright=nb["uright"], fv=nb["fv"])
        nm, m = oracle.search_for_triangulation(k1, k2, case["F12"][j], case["ep"][j], SF, SG, False, case["coarse"], case["check_orientation"])
        out.append((nm, m, has.copy()))
        a, b = ref["created_start"][j], ref["created_start"][j + 1]
        has[ref["idx1"][a:b]] = 1
    return out


def tags(case, ref):
    t = set()
    n = len(case["neighbours"])
    if n == 0:
        t.add("no_neighbours")
    if any(len(nb["fv"][0]) == 0 for nb in case["neighbours"]):
        t.add("empty_fv")
    if len(case["kf1"]["desc"]) > 1024:
        t.add("n1_strided")
    for pair, i1, i2, route, result, st in ref["trace"]:
        if result == 0:
            t.add("created:" + ROUTES[route])
        elif result == 1:
            t.add("route:low_parallax")
        elif result in (6, 7):
            side = st & 1 if result == 6 else st & 2
            t.add(f"reproj{result - 5}:" + ("stereo" if side else "mono"))
        else:
            t.add(RESULTS[result])
        if route == 3 and st == 3:
            t.add("route:stereo2_both_stereo")
    for j in range(n):
        a, b = ref["created_start"][j], ref["created_start"][j + 1]
        if len(np.unique(ref["idx2"][a:b])) < b - a:
            t.add("duplicate_idx2")
    if n >= 2:
        carried = search_with_carried(case, ref)
        kf1 = case["kf1"]
        for j in range(1, n):
            nm, m, has = carried[j]
            claimed = has.astype(bool) & ~kf1["has_mp"].astype(bool)
            k1 = dict(desc=kf1["desc"], keys=kf1["keys_un"], has_mp=kf1["has_mp"], uright=kf1["uright"], fv=kf1["fv"])
            nb = case["neighbours"][j]
            k2 = dict(desc=nb["desc"], keys=nb["keys_un"], has_mp=nb["has_mp"], uright=nb["uright"], fv=nb["fv"])
            _, m0 = oracle.search_for_triangulation(k1, k2, case["F12"][j], case["ep"][j], SF, SG, False, case["coarse"], case["check_orientation"])
            if (claimed & (m0 >= 0)).any():
                t.add("claimed_then_absent")
            if ((m0 != m) & ~claimed).any():
                t.add("hist_changed")
    return t

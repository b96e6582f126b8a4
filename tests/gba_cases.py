"""Seeded global-BA graphs at the edges of rgbl_global_bundle_adjustment (csrc/api_ba.cu, csrc/ba_factor.cu), shared by the emulated
(test_cuda_emu_gba.py) and the device (test_gpu_gba.py) tests, with the oracle (tests/gba_oracle.cpp) and the comparison against it.

Every case is a dict(name, problem, expect) like ba_cases.py's; `problem` adds `robust` and `stop` to the arguments, and `expect` names what
the case exists to reach, which check_coverage asserts on the problem and on the oracle's trace.  The graphs are loop-closed trajectories
(loop_graph): key frames on a circle looking outwards, every point seen by 3-10 consecutive key frames, the last key frames seeing the
points of the first.

Seeds: a loop held by one fixed key frame can be ill-conditioned; seeds 800 + 64 and 800 + 65, for one, move the oracle's own result by
4e-5 and 4e-4 when every input point moves by one float32 ulp, and there device and oracle legitimately part.  The seeds here were chosen
so that this move stays below SENSITIVITY (test_cuda_emu_gba.py checks it), which leaves the bars below room for the float32 rounding of
translations up to 60 m.

Bars (compare), those of ba_cases.compare without the erase flags: a case whose every decision margin in the trace exceeds 1e-6 must give
the oracle's iteration count and poses / points within 1e-5; any other case the iteration count and 1e-4.  Fixed key frames and points
without edges come back bit for bit."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile
from pathlib import Path

import numpy as np

import ba_cases as BC
from ba_dense_reference import _quat
from pose_cases import qmul, qrot, quat

HERE = Path(__file__).resolve().parent
CAM = BC.CAM
EXACT_MARGIN = BC.EXACT_MARGIN
TILE = 64                                # ba_factor.cuh kTile
SINGLE_CTA_MAX_OPT = 64                  # kSingleCtaMaxOpt (rgbl_kernels.h): above it the tiled path
MAX_FREE = 4096                          # RGBL_GBA_MAX_FREE_POSES


SENSITIVITY = 5e-5


def sensitivity(p):
    """The largest move of the oracle's poses / points when every input point moves up by one float32 ulp."""
    a = reference(p)
    b = reference(dict(p, points=np.nextafter(p["points"], np.float32(np.inf))))
    return max(float(np.abs(a[0].astype(np.float64) - b[0]).max()), float(np.abs(a[1].astype(np.float64) - b[1]).max()))


def solver_path(n_opt):
    return "single_cta" if n_opt <= SINGLE_CTA_MAX_OPT else "tiled"


def tiled_shape(n):
    """The launch shape of the tiled path at an n x n system: one tile or several, the last one full or partial."""
    return ("one_tile" if n <= TILE else "tiles", "full" if n % TILE == 0 else "partial")


# ---------------------------------------------------------------------------------------------------------------------------
# oracle: tests/gba_oracle.cpp (which includes oracle/ba_oracle.cpp), compiled into a temporary directory keyed by its sources
_olib = None


def _oracle_lib():
    global _olib
    if _olib is None:
        srcs = [HERE / "gba_oracle.cpp", HERE.parent / "oracle" / "ba_oracle.cpp", HERE.parent / "oracle" / "g2o_se3.inc"]
        key = hashlib.sha1(b"".join(s.read_bytes() for s in srcs)).hexdigest()[:12]
        out = Path(tempfile.gettempdir()) / f"rgbl_gba_oracle_{os.getuid()}_{key}" / "libgba_oracle.so"
        if not out.exists():
            out.parent.mkdir(parents=True, exist_ok=True)
            tmp = out.with_suffix(f".{os.getpid()}.so")
            subprocess.run(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-fno-fast-math", "-Wno-unused-function", f"-I{HERE.parent / 'oracle'}",
                            "-shared", "-o", str(tmp), str(srcs[0])], check=True)
            os.replace(tmp, out)
        import oracle
        _olib = C.CDLL(str(out))
        vp, i, f = C.c_void_p, C.c_int, C.c_float
        _olib.orc_global_bundle_adjustment_trace.argtypes = [i, vp, vp, i, vp, i, vp, vp, vp, vp, vp, f, f, f, f, f, i, i, vp, vp, vp, vp,
                                                             C.POINTER(oracle.BATraceC)]
        _olib.orc_global_bundle_adjustment_trace.restype = i
    return _olib


def _c(a, dt, shape=None):
    a = np.ascontiguousarray(a, dt)
    return a.reshape(shape) if shape else a


def oracle_gba(poses, pose_fixed, points, e_point, e_pose, obs, stereo, inv_sigma2, fx, fy, cx, cy, bf, iterations=10, robust=False, stop=False):
    """-> (poses[n,7], points[m,3], iterations, chi2, trace) with the trace of oracle.local_bundle_adjustment_trace (no edge margins)"""
    import oracle
    L = _oracle_lib()
    poses = _c(poses, np.float32, (-1, 7)); pose_fixed = _c(pose_fixed, np.uint8); points = _c(points, np.float32, (-1, 3))
    e_point = _c(e_point, np.int32); e_pose = _c(e_pose, np.int32); obs = _c(obs, np.float32, (-1, 3)); stereo = _c(stereo, np.uint8)
    inv_sigma2 = _c(inv_sigma2, np.float32)
    po = np.empty_like(poses); pt = np.empty_like(points); chi = C.c_double(0); st = np.array([1 if stop else 0], np.uint8)
    ct, ci = 10 * iterations + 1, iterations + 1
    arr = dict(trial_lambda=np.zeros(ct), trial_rho=np.zeros(ct), trial_accepted=np.zeros(ct, np.uint8), trial_ok=np.zeros(ct, np.uint8),
               iter_qmax=np.zeros(ci, np.int32), iter_bad=np.zeros(ci, np.uint8), iter_margin=np.full(ci, np.inf), edge_margin=np.full(1, np.inf))
    tr = oracle.BATraceC(ct, ci, *[a.ctypes.data for a in arr.values()])
    p = lambda a: a.ctypes.data
    it = L.orc_global_bundle_adjustment_trace(len(poses), p(poses), p(pose_fixed), len(points), p(points), len(e_point), p(e_point), p(e_pose), p(obs),
                                              p(stereo), p(inv_sigma2), fx, fy, cx, cy, bf, iterations, int(robust), p(st), p(po), p(pt), C.byref(chi),
                                              C.byref(tr))
    trace = {name: getattr(tr, name) for name, t in oracle.BATraceC._fields_ if t is not C.c_void_p and not name.startswith("cap_")}
    for name, a in arr.items():
        if name != "edge_margin":
            n = tr.n_trials if name.startswith("trial_") else tr.n_iters
            trace[name] = a[:n].astype(bool) if a.dtype == np.uint8 else a[:n]
    return po, pt, it, chi.value, trace


# ---------------------------------------------------------------------------------------------------------------------------
def loop_graph(seed, n_kf, n_fixed=1, n_pts=None, stereo_frac=0.5, noise=0.5, outlier_frac=0.02, pose_noise=(0.002, 0.02), point_noise=0.05,
               levels=8, iterations=10, robust=False, radius=None):
    """A loop-closed trajectory: n_kf key frames on a circle (radius `radius`, by default 0.3 n_kf m: one key frame every ~1.9 m) in the
    x-z plane looking outwards, key frame 0 first; key frames 0..n_fixed-1 fixed.  Each point lies 10-30 m outside the circle and is seen
    by up to 10 consecutive key frames, at least 3 unless the loop is shorter (indices modulo n_kf, so the last key frames see points of
    the first), each at a depth of more than 2 m.  Pixel noise `noise` x 1.2^level,
    information 1.2^-2 level, `outlier_frac` of the edges 15-60 px off; free poses start `pose_noise` (rad, m) and points
    `point_noise` (m) from the truth."""
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy, bf = CAM
    R = 0.3 * n_kf if radius is None else radius
    n_pts = n_pts or 6 * n_kf
    th = 2 * np.pi * np.arange(n_kf) / n_kf
    true_poses = np.empty((n_kf, 7))
    Rcw = []
    for k in range(n_kf):
        c, s = np.cos(th[k]), np.sin(th[k])
        Rk = np.array([[s, 0, -c], [0, 1, 0], [c, 0, s]])                       # rows: camera x, y, z (z = outwards)
        Rcw.append(Rk)
        q = _quat(Rk.astype(np.longdouble)).astype(np.float64)
        true_poses[k] = np.r_[q, -Rk @ np.array([R * c, 0.0, R * s])]
    true_poses = true_poses.astype(np.float32).astype(np.float64)
    true_poses[:, :4] /= np.linalg.norm(true_poses[:, :4], axis=1)[:, None]
    kk, jj, pts = [], [], []
    for j in range(n_pts):
        m = int(rng.integers(3, 11))
        k0 = int(rng.integers(n_kf))
        ks = [(k0 + i) % n_kf for i in range(min(m, n_kf))]
        phi = th[k0] + 0.5 * (len(ks) - 1) * 2 * np.pi / n_kf + rng.normal(0, 0.3) * 2 * np.pi / n_kf
        while True:
            d = rng.uniform(10, 30)
            P = np.array([(R + d) * np.cos(phi), rng.uniform(-3, 3), (R + d) * np.sin(phi)])
            seen = [k for k in ks if (Rcw[k] @ P + true_poses[k, 4:])[2] > 2.0]
            if len(seen) >= min(3, len(ks)):
                break
        ks = seen
        pts.append(P)
        kk += ks; jj += [j] * len(ks)
    pts = np.array(pts).astype(np.float32).astype(np.float64)
    kk, jj = np.array(kk), np.array(jj)
    o = rng.permutation(len(kk)); kk, jj = kk[o], jj[o]
    ne = len(kk)
    pc = np.array([qrot(true_poses[k, :4], pts[j]) + true_poses[k, 4:] for k, j in zip(kk, jj)]).reshape(ne, 3)
    sig = 1.2 ** rng.integers(0, levels, ne)
    u = fx * pc[:, 0] / pc[:, 2] + cx; v = fy * pc[:, 1] / pc[:, 2] + cy; ur = u - bf / pc[:, 2]
    obs = np.stack([u, v, ur], 1) + rng.normal(0, 1, (ne, 3)) * (noise * sig)[:, None]
    stereo = (rng.random(ne) < stereo_frac) & (obs[:, 2] >= 0)
    obs[~stereo, 2] = -1
    is_out = rng.random(ne) < outlier_frac
    obs[is_out, :2] += rng.choice([-1, 1], (int(is_out.sum()), 2)) * rng.uniform(15, 60, (int(is_out.sum()), 2))
    fixed = (np.arange(n_kf) < n_fixed).astype(np.uint8)
    poses = true_poses.copy()
    for k in np.nonzero(fixed == 0)[0]:
        poses[k, :4] = qmul(quat(rng.normal(0, 1, 3) * pose_noise[0]), poses[k, :4])
        poses[k, 4:] += rng.normal(0, 1, 3) * pose_noise[1]
    points = pts + rng.normal(0, 1, pts.shape) * point_noise
    return dict(poses=poses.astype(np.float32), pose_fixed=fixed, points=points.astype(np.float32), e_point=jj.astype(np.int32),
                e_pose=kk.astype(np.int32), obs=obs.astype(np.float32), stereo=stereo.astype(np.uint8), inv_sigma2=(1 / sig ** 2).astype(np.float32),
                cam=CAM, iterations=iterations, robust=robust, stop=False, true_poses=true_poses, true_points=pts, is_outlier=is_out)


def case(name, p, **expect):
    return dict(name=name, problem=p, expect=expect)


def _drop_edges(p, keep):
    for k in ("e_point", "e_pose", "obs", "stereo", "inv_sigma2", "is_outlier"):
        p[k] = p[k][keep]
    return p


def _plane(p, k):
    """Key frame k at the identity and a point at z = 0 seen by key frame k alone: its Jacobians are not finite, so neither is the (k, k)
    block of the reduced system, and every factorisation fails there."""
    j = int(p["e_point"][0])
    keep = p["e_point"] != j
    p = _drop_edges(p, keep)
    p["poses"][k] = [0, 0, 0, 1, 0, 0, 0]
    p["points"][j] = [1.5, -0.5, 0.0]
    ne = dict(e_point=[j], e_pose=[k], obs=[[CAM[2], CAM[3], -1]], stereo=[0], inv_sigma2=[1.0], is_outlier=[False])
    for key, v in ne.items():
        p[key] = np.concatenate([p[key], np.array(v, p[key].dtype)])
    return p


def _all_stereo(p):
    """Only the stereo edges (an observation whose right coordinate would be negative cannot be stereo)."""
    return _drop_edges(p, p["stereo"] != 0)


def selection():
    """n_opt 64 (the one-CTA kernel) and 65 (the first tiled system)."""
    return [case(f"sel{n}", loop_graph(801 + n, n + 1), n_opt=n, path=solver_path(n)) for n in (64, 65)]


def tiles():
    """Free-pose counts whose n = 6 n_opt lands on a tile multiple (96: 9 tiles) and one key frame either side, and 128 (12 tiles)."""
    return [case(f"tiles{n}", loop_graph(820 + n, n + 1), n_opt=n, path="tiled", shape=tiled_shape(6 * n)) for n in (95, 96, 97, 128)]


def loop200():
    return [case("loop200", loop_graph(900, 201, n_pts=1000), n_opt=200, path="tiled")]


def options():
    """Robust on and off, all-mono (two fixed key frames: the scale of a mono graph is not observable) and all-stereo, iterations 0 / 1 / 10,
    all on the tiled path."""
    out = [case("robust_on", loop_graph(910, 71, outlier_frac=0.05, robust=True), robust=True, huber=True),
           case("robust_off", loop_graph(910, 71, outlier_frac=0.05, robust=False), robust=False),
           case("mono", loop_graph(911, 72, n_fixed=2, stereo_frac=0.0), stereo_frac=0.0),
           case("stereo", _all_stereo(loop_graph(912, 71, stereo_frac=1.0)), stereo_frac=1.0)]
    for it in (0, 1, 10):
        out.append(case(f"iters{it}", loop_graph(920 + it, 70, iterations=it, robust=True), iterations_run=it if it < 10 else None))
    return out


def shapes():
    """Only the initial key frame fixed, a free key frame without edges, points without edges."""
    out = [case("init_only_fixed", loop_graph(936, 80), n_fixed=1)]
    p = loop_graph(931, 80)
    _drop_edges(p, p["e_pose"] != 40)
    out.append(case("free_no_edges", p, free_no_edge_pose=40, path="tiled"))
    p = loop_graph(932, 70)
    _drop_edges(p, ~np.isin(p["e_point"], [3, 17, 200]))
    out.append(case("points_no_edges", p, no_edge_points=[3, 17, 200]))
    return out


def failures():
    """Factorisations that fail on the tiled path: H = 0 (every information 0: lambda = 0 and the first pivot is 0), a point on the camera
    plane of a key frame in the middle of the system, and one of the last free key frame (the first bad pivot lies in the last tile)."""
    z = loop_graph(940, 80)
    z["inv_sigma2"][:] = 0
    return [case("allzero", z, solver_failures=10, unchanged=True, path="tiled"),
            case("plane", _plane(loop_graph(941, 80), 30), solver_failures=10, unchanged=True, path="tiled"),
            case("plane_last", _plane(loop_graph(942, 80), 79), solver_failures=10, unchanged=True, path="tiled", last_tile_pose=79)]


def stopped():
    """The stop flag raised before the call: no iteration, the inputs come back."""
    p = loop_graph(950, 70)
    p["stop"] = True
    return [case("stop_before", p, iterations_run=0, unchanged=True)]


def all_cases():
    return selection() + tiles() + loop200() + options() + shapes() + failures() + stopped()


def emulated_cases():
    """The subset that runs at one OS thread per CUDA thread: the first tiled system (65 free key frames, 2 iterations), a failure on the
    tiled path and the stop flag."""
    c = selection()[1]
    c["problem"]["iterations"] = 2
    return [c] + [x for x in failures() if x["name"] == "plane_last"] + stopped()


def refused(n_free=MAX_FREE + 1):
    """n_free free key frames and one fixed one, one point seen by all: more than RGBL_GBA_MAX_FREE_POSES."""
    n = n_free + 1
    poses = np.tile(np.array([0, 0, 0, 1, 0, 0, 0], np.float32), (n, 1))
    return dict(poses=poses, pose_fixed=(np.arange(n) == 0).astype(np.uint8), points=np.array([[0, 0, 10]], np.float32),
                e_point=np.zeros(n, np.int32), e_pose=np.arange(n, dtype=np.int32), obs=np.tile(np.array([CAM[2], CAM[3], -1], np.float32), (n, 1)),
                stereo=np.zeros(n, np.uint8), inv_sigma2=np.ones(n, np.float32), cam=CAM, iterations=10, robust=False, stop=False)


def args(p):
    return (p["poses"], p["pose_fixed"], p["points"], p["e_point"], p["e_pose"], p["obs"], p["stereo"], p["inv_sigma2"], *p["cam"])


def reference(p):
    """-> (poses, points, iterations, trace)"""
    po, pt, it, _, tr = oracle_gba(*args(p), iterations=p["iterations"], robust=p["robust"], stop=p["stop"])
    return po, pt, it, tr


def qualifies(trace):
    return min(trace["min_rho_margin"], trace["min_stop_margin"], trace["min_huber_margin"]) > EXACT_MARGIN


def check_coverage(c, trace):
    e, p, name = c["expect"], c["problem"], c["name"]
    free = p["pose_fixed"] == 0
    n_opt = int(free.sum())
    if "n_opt" in e:
        assert n_opt == e["n_opt"], name
    if "path" in e:
        assert solver_path(n_opt) == e["path"], (name, n_opt)
    if "shape" in e:
        assert tiled_shape(6 * n_opt) == e["shape"], name
    if "robust" in e:
        assert p["robust"] == e["robust"], name
    if e.get("huber"):
        assert trace["min_huber_margin"] < np.inf and p["is_outlier"].any(), name
    if "stereo_frac" in e:
        assert p["stereo"].mean() == e["stereo_frac"], name
    if e.get("iterations_run") is not None:
        assert trace["n_iters"] == e["iterations_run"], (name, trace["n_iters"])
    if "n_fixed" in e:
        assert int((~free).sum()) == e["n_fixed"] and not free[0], name
    if "free_no_edge_pose" in e:
        k = e["free_no_edge_pose"]
        assert free[k] and not (p["e_pose"] == k).any(), name
    if "no_edge_points" in e:
        assert not np.isin(p["e_point"], e["no_edge_points"]).any(), name
    if "solver_failures" in e:
        assert trace["solver_failures"] >= e["solver_failures"] and not trace["trial_ok"].any(), (name, trace)
    if "last_tile_pose" in e:
        slot = int(np.cumsum(free)[e["last_tile_pose"]] - 1)
        assert 6 * slot >= (6 * n_opt - 1) // TILE * TILE, name                   # its block lies in the last tile
        j = int(p["e_point"][-1])                                                   # the point on the camera plane (_plane) touches no other block
        assert p["points"][j, 2] == 0 and set(p["e_pose"][p["e_point"] == j].tolist()) == {e["last_tile_pose"]}, name


def compare(c, got, ref):
    """got = (poses, points, iterations) of the device, ref = reference(problem) -> (bar, d_pose, d_point)"""
    gpo, gpt, git = got
    rpo, rpt, rit, trace = ref
    p, name = c["problem"], c["name"]
    fixed = p["pose_fixed"] != 0
    assert gpo[fixed].tobytes() == p["poses"][fixed].tobytes(), name
    no_edge = np.bincount(p["e_point"], minlength=len(gpt)) == 0
    assert gpt[no_edge].tobytes() == p["points"][no_edge].tobytes(), name
    if c["expect"].get("unchanged"):
        assert np.array_equal(rpt, p["points"]) and gpo.tobytes() == rpo.tobytes() and gpt.tobytes() == rpt.tobytes(), name
    assert np.isfinite(gpo).all() and np.isfinite(gpt).all(), name
    assert git == rit, (name, git, rit)
    d_pose = float(np.abs(gpo.astype(np.float64) - rpo).max()) if len(gpo) else 0.0
    d_pt = float((np.abs(gpt.astype(np.float64) - rpt) / np.maximum(1.0, np.abs(rpt))).max()) if len(gpt) else 0.0
    bar, tol = ("exact", 1e-5) if qualifies(trace) else ("loose", 1e-4)
    assert d_pose < tol and d_pt < tol, (name, bar, d_pose, d_pt)
    return bar, d_pose, d_pt


def dense_case():
    """70 free key frames, few points, one iteration whose first trial is accepted, robust: for gba_dense_reference.lm_step.  On a circle
    of 3 m, so that the float32 rounding of the translations stays well below the reference's 1e-6."""
    return case("dense70", loop_graph(960, 71, n_pts=110, iterations=1, robust=True, outlier_frac=0.05, radius=3.0), first_accepted=True, path="tiled")


def check_first_accepted(c, trace):
    assert trace["trial_accepted"][0] and trace["n_iters"] == 1, (c["name"], trace)

"""Seeded local-BA graphs at the edges of rgbl_local_bundle_adjustment (csrc/api_ba.cu), shared by the emulated (test_cuda_emu_ba.py) and
the device (test_gpu_ba_edges.py) tests, with the comparison against oracle.local_bundle_adjustment_trace.

Every case is a dict(name, family, problem, expect): `problem` holds the arguments of the call (poses, pose_fixed, points, edges, cam,
iterations) plus the generating `true_poses` / `true_points` and `exact_truth` (noise- and outlier-free: the optimum IS the truth);
`expect` names what the case exists to reach - graph shapes (checked on the problem) and LM paths (checked on the oracle's trace) - and
`check_coverage` asserts them, so a generator change cannot silently stop covering a path.

Bars (compare): a case whose every decision margin in the trace exceeds 1e-6 (relative) must match the oracle exactly: identical iteration
count and erase flags, poses within 1e-5 and points within 1e-5 max(1, |p|).  Any other case keeps the bar of test_gpu_ba.py: 1e-4, and
flags that differ only on edges whose own margin is below the limit.

Paths no legitimate input reaches in one call, so no case forces them:
  * a successful factorisation after a failed one.  With lambda > 0 the reduced system is H_pp + lambda I minus a Schur term that leaves it
    positive definite by lambda = at least 1e-5 3^-10 max|diag H|, ten orders above the rounding of its entries; a pivot fails only when
    H = 0 (then lambda = 0 and stays 0: `allzero`) or when H is not finite (a point on a camera plane: `plane`), and both persist for
    every trial of the call.  What a recovery would exercise - the status word, S and x_p written by a failed solve and reused by the next -
    is reached across calls instead: test_gpu_ba_edges.py runs a well-posed graph after a failing one on the same context.
  * qmax == 10 through ten finite rejected trials.  The damping grows by 2^45 over them, so the tenth step is a vanishing gradient step
    that lowers chi2 unless the estimate already is the minimum to rounding; a search over seeds, start distances, outlier shares and
    noise-free graphs started at their truth found runs of up to 6.  qmax == 10, and with it a call whose last evaluated trial was
    rejected, is reached through ten failed factorisations (`allzero`); `plane` ends on a rejected trial whose rho is not a number."""
import numpy as np

import oracle
from orb_slam3_rgbl_b200 import synthetic as S
from pose_cases import qmul, qrot, quat

CAM = (S.KITTI_FX, S.KITTI_FY, S.KITTI_CX, S.KITTI_CY, S.KITTI_BF)
EXACT_MARGIN = 1e-6

# ba_cholesky_kernel's launch (api_ba.cu, rgbl_local_bundle_adjustment): S and y are staged in shared memory when
# (n * n + n) * sizeof(double) <= 200 KiB, and the CTA has 256 threads up to n = 192, 1024 above.  n = 6 n_opt.
CHOL_SMEM_BYTES = 200 * 1024
CHOL_SMALL_N = 192


def cholesky_shape(n_opt):
    n = 6 * n_opt
    return ("shared" if (n * n + n) * 8 <= CHOL_SMEM_BYTES else "global", 256 if n <= CHOL_SMALL_N else 1024)


# seeds found by searching with the oracle's trace for the paths each lm case names, every decision margin above 1e-6, and a result that
# moves by less than 1e-6 when every input point moves by one float32 ulp, then frozen.  The last condition matters: a start this far
# off can carry an edge to within millimetres of a camera plane, where the normal equations amplify rounding by ten orders and device and
# oracle legitimately part (seed 1096 of the first setting does, at |z| = 0.006 m after its first step).
SEED = {"rejects0": 1136, "rejects1": 1076, "rejects2": 1071, "nbad": 1000}


def graph(seed, n_fixed, n_free, vis, stereo_frac=0.6, noise=0.6, outlier_frac=0.0, pose_noise=(0.004, 0.03), point_noise=0.06, levels=8,
          bf=CAM[4], iterations=10, shuffle=True):
    """A local-BA graph.  vis[k, j]: key frame k sees point j, with the fixed key frames in rows 0..n_fixed-1; with `shuffle` the key
    frames are then placed in random order (fixed ones anywhere) and the edges listed in random order.  Key frames sit within 2 m of each
    other looking down +z at points 10-45 m away; pixel noise sigma `noise` x 1.2^level, information 1.2^-2 level; `outlier_frac` of the
    edges are 15-60 px off; free poses start `pose_noise` (rad, m) and points `point_noise` (m) from the truth, which is rounded to
    float32 first, so a noise-free graph started with zero noise starts at its optimum."""
    rng = np.random.default_rng(seed)
    fx, fy, cx, cy, _ = CAM
    vis = np.asarray(vis, bool)
    n_kf, n_pts = n_fixed + n_free, vis.shape[1]
    assert vis.shape[0] == n_kf
    order = rng.permutation(n_kf) if shuffle else np.arange(n_kf)                    # array position -> logical key frame
    vis = vis[order]
    fixed = (order < n_fixed).astype(np.uint8)
    true_poses = np.empty((n_kf, 7))
    for k in range(n_kf):
        q = quat(rng.normal(0, 0.02, 3))
        c = np.array([rng.uniform(-2, 2), rng.uniform(-0.3, 0.3), rng.uniform(0, 3)])
        true_poses[k] = np.r_[q, -qrot(q, c)]
    true_poses = true_poses.astype(np.float32).astype(np.float64)
    true_poses[:, :4] /= np.linalg.norm(true_poses[:, :4], axis=1)[:, None]          # what the call makes of the float32 quaternion
    z = rng.uniform(10, 45, n_pts)
    pts = np.stack([rng.uniform(-0.45, 0.45, n_pts) * z, rng.uniform(-0.12, 0.1, n_pts) * z, z], 1).astype(np.float32).astype(np.float64)
    kk, jj = np.nonzero(vis)
    if shuffle:
        o = rng.permutation(len(kk)); kk, jj = kk[o], jj[o]
    ne = len(kk)
    pc = np.array([qrot(true_poses[k, :4], pts[j]) + true_poses[k, 4:] for k, j in zip(kk, jj)]).reshape(ne, 3)
    sig = 1.2 ** rng.integers(0, levels, ne)
    u = fx * pc[:, 0] / pc[:, 2] + cx; v = fy * pc[:, 1] / pc[:, 2] + cy; ur = u - bf / pc[:, 2]
    obs = np.stack([u, v, ur], 1) + rng.normal(0, 1, (ne, 3)) * (noise * sig)[:, None]
    stereo = (rng.random(ne) < stereo_frac) & (obs[:, 2] >= 0)                       # a stereo observation has mvuRight >= 0
    obs[~stereo, 2] = -1
    is_out = rng.random(ne) < outlier_frac
    obs[is_out, :2] += rng.choice([-1, 1], (int(is_out.sum()), 2)) * rng.uniform(15, 60, (int(is_out.sum()), 2))
    poses = true_poses.copy()
    for k in np.nonzero(fixed == 0)[0]:
        poses[k, :4] = qmul(quat(rng.normal(0, 1, 3) * pose_noise[0]), poses[k, :4])
        poses[k, 4:] += rng.normal(0, 1, 3) * pose_noise[1]
    points = pts + rng.normal(0, 1, pts.shape) * point_noise
    return dict(poses=poses.astype(np.float32), pose_fixed=fixed, points=points.astype(np.float32), e_point=jj.astype(np.int32),
                e_pose=kk.astype(np.int32), obs=obs.astype(np.float32), stereo=stereo.astype(np.uint8), inv_sigma2=(1 / sig ** 2).astype(np.float32),
                cam=(*CAM[:4], bf), iterations=iterations, true_poses=true_poses, true_points=pts, is_outlier=is_out,
                exact_truth=noise == 0 and outlier_frac == 0)


def vis_degree(seed, n_fixed, n_free, n_pts, deg, min_pose_edges=12):
    """Every point seen by `deg` key frames, at least one of them free; every free key frame sees at least `min_pose_edges` points."""
    rng = np.random.default_rng(seed + 7919)
    n_kf = n_fixed + n_free
    vis = np.zeros((n_kf, n_pts), bool)
    for j in range(n_pts):
        vis[n_fixed + rng.integers(n_free), j] = True
        rest = np.nonzero(~vis[:, j])[0]
        vis[rng.choice(rest, min(deg, n_kf) - 1, replace=False), j] = True
    for k in range(n_fixed, n_kf):
        short = min_pose_edges - int(vis[k].sum())
        if short > 0:
            vis[k, rng.choice(np.nonzero(~vis[k])[0], short, replace=False)] = True
    return vis


def case(name, family, p, **expect):
    return dict(name=name, family=family, problem=p, expect=expect)


def solver(sizes=(1, 26, 27, 32, 33, 64), n_pts=160, iterations=10):
    """The three launches of ba_cholesky_kernel: shared memory with 256 threads up to 26 free key frames, global memory (factored in
    place, y aliased onto x) from 27, and 1024 threads from 33."""
    return [case(f"solver{n}", "solver", graph(100 + n, 2, n, vis_degree(100 + n, 2, n, max(n_pts, 4 * n), 5), iterations=iterations), n_opt=n)
            for n in sizes]


def degree(many=3000, iterations=10):
    """Point degrees around the 32 lanes of ba_schur_kernel's two loops, points nothing free sees, and free key frames with edge counts
    around ba_pose_sum_kernel's 256-thread stride."""
    n_fixed, n_free, fill = 3, 45, 150
    degs = [1, 1, 2, 31, 32, 33, 40, 48]
    vis = np.zeros((48, len(degs) + 2 + fill), bool)
    rng = np.random.default_rng(200)
    for j, m in enumerate(degs):
        vis[rng.choice(np.arange(n_fixed, 48), min(m, n_free), replace=False), j] = True
        if m > n_free:
            vis[:n_fixed, j] = True
    vis[:n_fixed, len(degs)] = True                          # seen by the fixed key frames only; the next point has no edge at all
    vis[:, len(degs) + 2:] = vis_degree(201, n_fixed, n_free, fill, 5)
    p = graph(202, n_fixed, n_free, vis, shuffle=False, iterations=iterations)
    k0, k1 = [np.nonzero(p["e_point"] == j)[0][0] for j in (0, 1)]
    p["stereo"][k0] = 0; p["obs"][k0, 2] = -1                # point 0: one mono observation (H_ll of rank 2), point 1: one stereo
    p["stereo"][k1] = 1; p["obs"][k1, 2] = max(p["obs"][k1, 2], p["obs"][k1, 0] - 30)
    out = [case("deg_points", "degree", p, point_degrees=[1, 2, 31, 32, 33, 40, 48], fixed_only_point=len(degs), no_edge_point=len(degs) + 1)]
    want = [0, 1, 255, 256, 257] + ([many] if many else [])
    n_pts = max(want) + 40
    vis = np.zeros((2 + len(want) + 2, n_pts), bool)
    vis[:2] = True                                           # two fixed key frames see every point
    rng = np.random.default_rng(203)
    for i, m in enumerate(want):
        vis[2 + i, rng.choice(n_pts, m, replace=False)] = True
    vis[-2:] = rng.random((2, n_pts)) < 0.5
    out.append(case("deg_poses" if many else "deg_poses_small", "degree", graph(204, 2, len(want) + 2, vis, iterations=iterations), pose_degrees=want))
    return out


def grid():
    """n_edges, n_points and n_poses one below, at and one above the 128-thread CTAs of the per-edge, per-point and per-pose kernels (a
    last CTA with 127 idle threads, block_sum_to over partial warps), and 140 key frames of which 120 are fixed."""
    out = []
    for x in (127, 128, 129):
        vis = vis_degree(300 + x, 2, 5, 36, 4)
        kk, jj = np.nonzero(vis)
        assert len(kk) >= x
        rng = np.random.default_rng(310 + x)
        for i in rng.permutation(len(kk)):                   # thin to exactly x edges, keeping two observations of every point
            if vis.sum() > x and vis[:, jj[i]].sum() > 2:
                vis[kk[i], jj[i]] = False
        out.append(case(f"grid_e{x}", "grid", graph(320 + x, 2, 5, vis), n_edges=x))
        out.append(case(f"grid_p{x}", "grid", graph(330 + x, 2, 6, vis_degree(330 + x, 2, 6, x, 4)), n_points=x))
        out.append(case(f"grid_q{x}", "grid", graph(340 + x, x - 9, 9, vis_degree(340 + x, x - 9, 9, 120, 6)), n_poses=x))
    out.append(case("grid_q140", "grid", graph(350, 120, 20, vis_degree(350, 120, 20, 200, 6)), n_poses=140))
    return out


def lm():
    """The LM control flow: runs of rejected trials followed by an accepted one (the ping-pong of the two state buffers), n_bad >= 3,
    rho == 0, factorisations that fail up to qmax == 10, calls whose last evaluated trial was rejected (the erase flags then come from
    the errors of a state that was not kept), and iterations 0, 1 and 2."""
    def hard(seed, **kw):
        return graph(seed, 2, 6, vis_degree(seed, 2, 6, 120, 5), **kw)
    far = dict(outlier_frac=0.4, pose_noise=(0.5, 2.5), point_noise=2.0)
    out = [case("rejects0", "lm", hard(SEED["rejects0"], **far), reject_run=6, accept_after_reject=True),
           case("rejects1", "lm", hard(SEED["rejects1"], **far), reject_run=5, accept_after_reject=True),
           case("rejects2", "lm", hard(SEED["rejects2"], **far), reject_run=3, accept_after_reject=True),
           case("nbad", "lm", hard(SEED["nbad"], outlier_frac=0.3, pose_noise=(0.3, 1.5), point_noise=1.0), nbad=True)]
    # rho == 0: points on the optical axis of two key frames that differ by a translation along it, observed at (cx, cy) exactly: every
    # error is 0, so b = 0, the step is 0 and chi2 stays 0
    n = 12
    ax = dict(poses=np.array([[0, 0, 0, 1, 0, 0, 0], [0, 0, 0, 1, 0, 0, -1.0]], np.float32), pose_fixed=np.array([1, 0], np.uint8),
              points=np.stack([np.zeros(n), np.zeros(n), np.arange(5.0, 5 + n)], 1).astype(np.float32),
              e_point=np.tile(np.arange(n), 2).astype(np.int32), e_pose=np.repeat([0, 1], n).astype(np.int32),
              obs=np.tile(np.array([CAM[2], CAM[3], -1], np.float32), (2 * n, 1)), stereo=np.zeros(2 * n, np.uint8),
              inv_sigma2=np.ones(2 * n, np.float32), cam=CAM, iterations=10, exact_truth=False)
    out.append(case("rho0", "lm", ax, rho0=True, ends_rejected=True, iterations_run=1))
    # H = 0: every information value 0, so lambda = 0 and the first pivot is 0 in all ten trials
    z = hard(400)
    z["inv_sigma2"][:] = 0
    z["exact_truth"] = False
    out.append(case("allzero", "lm", z, solver_failures=10, qmax=True, ends_rejected=True, unchanged=True))
    # a point on the camera plane of a free key frame (z = 0 exactly: the identity pose and a point with z = 0): its Jacobians are not
    # finite, so neither is H and every factorisation fails
    pl = hard(401, shuffle=False)
    k = int(pl["e_pose"][np.nonzero(pl["pose_fixed"][pl["e_pose"]] == 0)[0][0]])
    j = int(pl["e_point"][np.nonzero(pl["e_pose"] == k)[0][0]])
    pl["poses"][k] = [0, 0, 0, 1, 0, 0, 0]
    pl["points"][j] = [1.5, -0.5, 0.0]
    pl["exact_truth"] = False
    out.append(case("plane", "lm", pl, solver_failures=10, ends_rejected=True, unchanged=True))
    for it in (0, 1, 2):
        out.append(case(f"iters{it}", "lm", hard(410 + it, outlier_frac=0.05, iterations=it), iterations_run=it))
    return out


def numeric():
    """Input quaternions with qw < 0 and norms away from 1 (ba_init_state_kernel; fixed key frames must come back bit for bit), all-mono
    and all-stereo graphs, stereo with bf = 0, points behind a camera, a noise-free graph started at the truth (steps with
    theta^2 < 1e-10 in se3_exp) and one started 0.5 rad away."""
    def g(seed, **kw):
        return graph(seed, 2, 6, vis_degree(seed, 2, 6, 150, 5), **kw)
    out = []
    p = g(500, outlier_frac=0.03)
    s = np.random.default_rng(501).choice([-1.0, 1.0], len(p["poses"])) * np.random.default_rng(502).uniform(0.5, 2.0, len(p["poses"]))
    s[:2] = [-1.0, -1.7]
    p["poses"][:, :4] *= s[:, None].astype(np.float32)
    out.append(case("quat", "numeric", p, negative_qw=True))
    out.append(case("mono", "numeric", g(510, stereo_frac=0.0, outlier_frac=0.03)))
    out.append(case("stereo", "numeric", g(511, stereo_frac=1.0, outlier_frac=0.03)))
    out.append(case("stereo_bf0", "numeric", g(512, stereo_frac=1.0, outlier_frac=0.03, bf=0.0)))
    p = g(513, outlier_frac=0.03, shuffle=False)
    for j in (0, 1, 2):                                      # the observations say in front, the start says 3-5 m behind
        p["points"][j, 2] = -3.0 - j
    out.append(case("behind", "numeric", p, behind_points=(0, 1, 2)))
    out.append(case("at_truth", "numeric", g(514, noise=0.0, pose_noise=(0, 0), point_noise=0.0)))
    out.append(case("noise_free", "numeric", g(515, noise=0.0)))
    out.append(case("far_rotation", "numeric", g(516, noise=0.0, pose_noise=(0.3, 0.5), point_noise=0.3)))
    return out


def no_free_pose():
    """n_opt = 0: every key frame fixed (structure-only adjustment), with no reduced system and x_p never written."""
    return [case("all_fixed", "no_free_pose", graph(600, 5, 0, vis_degree(600, 4, 1, 100, 4), outlier_frac=0.03), n_opt=0),
            case("all_fixed_exact", "no_free_pose", graph(601, 4, 0, vis_degree(601, 3, 1, 60, 3), noise=0.0), n_opt=0)]


def dense():
    """Small graphs run for one iteration whose first trial is accepted, for ba_dense_reference.lm_step: all-mono, all-stereo, mixed with
    outliers (Huber weights below 1), a point seen by fixed key frames only, and a point of degree 33."""
    def g(seed, n_free=4, n_pts=40, vis=None, **kw):
        return graph(seed, 2, n_free, vis_degree(seed, 2, n_free, n_pts, 4, 3) if vis is None else vis, iterations=1, **kw)
    fo = vis_degree(703, 2, 4, 40, 4, 3)
    fo[:, 0] = [True, True, False, False, False, False]
    m33 = vis_degree(704, 2, 33, 40, 4, 3)
    m33[:, 0] = [False, False] + [True] * 33
    return [case("dense_mono", "dense", g(700, stereo_frac=0.0), first_accepted=True),
            case("dense_stereo", "dense", g(701, stereo_frac=1.0), first_accepted=True),
            case("dense_mixed", "dense", g(702, outlier_frac=0.2, pose_noise=(0.02, 0.1), point_noise=0.3), first_accepted=True, huber=True),
            case("dense_fixed_only", "dense", g(703, vis=fo, shuffle=False), first_accepted=True, fixed_only_point=0),
            case("dense_m33", "dense", g(704, n_free=33, vis=m33, shuffle=False), first_accepted=True, point_degrees=[33])]


FAMILIES = [solver, degree, grid, lm, numeric, no_free_pose, dense]


def all_cases():
    return [c for f in FAMILIES for c in f()]


def emulated_cases():
    """The subset that runs at one OS thread per CUDA thread: all three Cholesky launches (26, 27 and 33 free key frames, the 1024-thread
    one capped at 2 iterations), points of degree 33 and more and key frames with 0 to 257 edges (2 iterations), the grids at 129, rejected-then-accepted trials, both
    solver failures, rho == 0 and iterations = 0."""
    names = {"grid_e129", "grid_p129", "grid_q129", "rejects0", "rho0", "allzero", "plane", "iters0", "behind", "all_fixed"}
    return (solver((26, 27), 60, 3) + solver((33,), 60, 2) + degree(0, 2)
            + [c for c in all_cases() if c["name"] in names])


def args(p):
    return (p["poses"], p["pose_fixed"], p["points"], p["e_point"], p["e_pose"], p["obs"], p["stereo"], p["inv_sigma2"], *p["cam"], p["iterations"])


def reference(p):
    """-> (poses, points, erase, iterations, trace)"""
    po, pt, er, it, _, tr = oracle.local_bundle_adjustment_trace(*args(p))
    return po, pt, er, it, tr


def qualifies(trace):
    return trace["min_margin"] > EXACT_MARGIN


def check_coverage(c, trace):
    """The graph shapes and trace conditions the case exists to reach."""
    e, p, name = c["expect"], c["problem"], c["name"]
    free = p["pose_fixed"] == 0
    pdeg = np.bincount(p["e_point"], minlength=len(p["points"]))
    if "n_opt" in e:
        assert int(free.sum()) == e["n_opt"], name
    for m in e.get("point_degrees", []):
        assert ((pdeg == m) & (np.bincount(p["e_point"][free[p["e_pose"]]], minlength=len(pdeg)) == min(m, free.sum()))).any(), (name, m)
    if "fixed_only_point" in e:
        k = p["e_point"] == e["fixed_only_point"]
        assert k.any() and not free[p["e_pose"][k]].any(), name
    if "no_edge_point" in e:
        assert pdeg[e["no_edge_point"]] == 0, name
    if "pose_degrees" in e:
        have = np.bincount(p["e_pose"], minlength=len(free))[free]
        assert set(e["pose_degrees"]) <= set(have.tolist()), (name, sorted(have))
    for key, arr in (("n_edges", "e_point"), ("n_points", "points"), ("n_poses", "poses")):
        if key in e:
            assert len(p[arr]) == e[key], (name, key, len(p[arr]))
    if e.get("negative_qw"):
        assert (p["poses"][free, 3] < 0).any() and (p["poses"][~free, 3] < 0).any(), name
    if e.get("first_accepted"):
        assert trace["trial_accepted"][0] and trace["n_iters"] == 1, (name, trace)
    if e.get("huber"):
        assert trace["min_huber_margin"] < np.inf and int(p["is_outlier"].sum()) > 0, name
    if "reject_run" in e:
        assert trace["max_reject_run"] >= e["reject_run"], (name, trace)
    if e.get("accept_after_reject"):
        a = trace["trial_accepted"]
        assert any(not a[i] and not a[i + 1] and not a[i + 2] and a[i + 3] for i in range(len(a) - 3)), (name, a)
    if e.get("qmax"):
        assert trace["term_qmax"] and 10 in trace["iter_qmax"], (name, trace)
    if e.get("nbad"):
        assert trace["term_nbad"], (name, trace)
    if e.get("rho0"):
        assert trace["term_rho0"], (name, trace)
    if e.get("ends_rejected"):
        assert trace["ended_on_rejected_trial"], (name, trace)
    if "solver_failures" in e:
        assert trace["solver_failures"] >= e["solver_failures"] and not trace["trial_ok"].all(), (name, trace)
    if "iterations_run" in e:
        assert trace["n_iters"] == e["iterations_run"], (name, trace)


def compare(c, got, ref):
    """got / ref = (poses, points, erase, iterations) of the device / (.., trace) of the oracle.  -> (bar, d_pose, d_point) with the bar
    applied ('exact' or 'loose') and the largest pose and (relative) point differences."""
    gpo, gpt, ger, git = got
    rpo, rpt, rer, rit, trace = ref
    p, name = c["problem"], c["name"]
    fixed = p["pose_fixed"] != 0
    assert gpo[fixed].tobytes() == p["poses"][fixed].tobytes(), name                         # fixed key frames come back bit for bit
    no_edge = np.bincount(p["e_point"], minlength=len(gpt)) == 0
    assert gpt[no_edge].tobytes() == p["points"][no_edge].tobytes(), name                    # and so do points nothing observes
    if c["expect"].get("unchanged"):
        assert rpo.tobytes() == p["poses"].tobytes() and np.array_equal(rpt, p["points"]), name
    assert np.isfinite(gpo).all() and np.isfinite(gpt).all(), name
    d_pose = float(np.abs(gpo.astype(np.float64) - rpo).max())
    d_pt = float((np.abs(gpt.astype(np.float64) - rpt) / np.maximum(1.0, np.abs(rpt))).max())
    diff = ger != rer
    if qualifies(trace):
        bar, tol = "exact", 1e-5
        assert git == rit and not diff.any(), (name, git, rit, int(diff.sum()))
    else:
        bar, tol = "loose", 1e-4
        assert git == rit, (name, git, rit, trace)
        assert (trace["edge_margin"][diff] <= EXACT_MARGIN).all(), (name, np.nonzero(diff)[0], trace["edge_margin"][diff])
    assert d_pose < tol and d_pt < tol, (name, bar, d_pose, d_pt)
    if "behind_points" in c["expect"]:                                                       # flagged by the depth test
        j = list(c["expect"]["behind_points"])
        assert (gpt[j, 2] < 0).all() and ger[np.isin(p["e_point"], j)].all(), name
    return bar, d_pose, d_pt


def compare_dense(c, poses, points):
    """poses / points after one iteration against ba_dense_reference.lm_step -> the largest pose and (relative) point differences."""
    import ba_dense_reference as BD
    dpo, dpt = BD.lm_step(*args(c["problem"]))
    po = poses.astype(np.float64) * np.where(poses[:, 3:4] < 0, -1.0, 1.0)
    d_pose = float(np.abs(po - dpo).max())
    d_pt = float((np.abs(points - dpt) / np.maximum(1.0, np.abs(dpt))).max())
    assert d_pose < 1e-6 and d_pt < 1e-6, (c["name"], d_pose, d_pt)
    return d_pose, d_pt


def truth(c, poses, points):
    """Independent of the oracle: on a noise-free graph the result is the generating poses and points."""
    p = c["problem"]
    if not p["exact_truth"]:
        return None
    q = poses[:, :4].astype(np.float64) * np.sign(poses[:, 3:4]); q /= np.linalg.norm(q, axis=1)[:, None]
    seen = np.bincount(p["e_point"], minlength=len(points)) >= 2
    d_pose = max(float(np.abs(q - p["true_poses"][:, :4]).max()), float(np.abs(poses[:, 4:] - p["true_poses"][:, 4:]).max()))
    d_pt = float((np.abs(points - p["true_points"])[seen] / np.maximum(1.0, np.abs(p["true_points"][seen]))).max())
    assert d_pose < 5e-4 and d_pt < 5e-4, (c["name"], d_pose, d_pt)
    return d_pose, d_pt

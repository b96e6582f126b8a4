"""One Levenberg-Marquardt step of global bundle adjustment in numpy longdouble: ba_dense_reference.lm_step's definitions (central-difference
Jacobians, dense normal equations of all free key frames and points, lambda = 1e-5 max |H_ii|, a longdouble Cholesky), with the robust
kernel of Optimizer::BundleAdjustment as a choice: Huber with d^2 = 5.99 (mono) / 7.815 (stereo) when `robust`, else plain least squares
(weight 1)."""
import numpy as np

from ba_dense_reference import H_STEP, LD, _exp, _project, _quat, _rot, _solve_spd


def lm_step(poses, pose_fixed, points, e_point, e_pose, obs, stereo, inv_sigma2, fx, fy, cx, cy, bf, robust=False, d2_mono=5.99, d2_stereo=7.815):
    """The estimates after the first LM trial, taken as accepted -> (poses[n, 7] with qw >= 0, points[m, 3]) in longdouble; fixed key
    frames are returned as given."""
    cam = tuple(LD(float(v)) for v in (fx, fy, cx, cy, bf))
    q = np.asarray(poses, np.float64)[:, :4].astype(LD)
    q /= np.sqrt((q * q).sum(1))[:, None]
    Rs = [_rot(qi) for qi in q]
    ts = np.asarray(poses, np.float64)[:, 4:].astype(LD)
    P = np.asarray(points, np.float64).astype(LD)
    slot = np.cumsum(np.asarray(pose_fixed) == 0) - 1
    n_opt = int((np.asarray(pose_fixed) == 0).sum())
    n = 6 * n_opt + 3 * len(P)
    Hm = np.zeros((n, n), LD); g = np.zeros(n, LD)
    for k in range(len(e_point)):
        i, j, st = int(e_pose[k]), int(e_point[k]), bool(stereo[k])
        d = 3 if st else 2
        z = np.asarray(obs[k], np.float64).astype(LD)[:d]
        r = z - _project(Rs[i], ts[i], P[j], cam, st, True)
        s = LD(float(inv_sigma2[k])) * (r @ r)
        d2 = LD(d2_stereo) if st else LD(d2_mono)
        w = LD(1) if (not robust or s <= d2) else np.sqrt(d2 / s)
        J = np.zeros((d, 9), LD)
        for c in range(9):
            vals = []
            for sign in (1, -1):
                a = np.zeros(6, LD); b = np.zeros(3, LD)
                if c < 6:
                    a[c] = sign * H_STEP
                else:
                    b[c - 6] = sign * H_STEP
                dR, dt = _exp(a)
                vals.append(z - _project(dR @ Rs[i], dR @ ts[i] + dt, P[j] + b, cam, st, False))
            J[:, c] = (vals[0] - vals[1]) / (2 * H_STEP)
        idx = np.r_[np.arange(6 * slot[i], 6 * slot[i] + 6) if not pose_fixed[i] else np.zeros(0, int), 6 * n_opt + 3 * j + np.arange(3)]
        Jk = J[:, 9 - len(idx):]
        wi = w * LD(float(inv_sigma2[k]))
        Hm[np.ix_(idx, idx)] += wi * (Jk.T @ Jk)
        g[idx] -= wi * (Jk.T @ r)
    lam = LD(1e-5) * np.abs(np.diag(Hm)).max()
    x = _solve_spd(Hm + lam * np.eye(n, dtype=LD), g)
    out_poses = np.asarray(poses, np.float64).astype(LD).copy()
    for i in range(len(out_poses)):
        if pose_fixed[i]:
            continue
        dR, dt = _exp(x[6 * slot[i]:6 * slot[i] + 6])
        out_poses[i] = np.r_[_quat(dR @ Rs[i]), dR @ ts[i] + dt]
    return out_poses, P + x[6 * n_opt:].reshape(-1, 3)


def compare(p, poses, points, tol=1e-6):
    """poses / points after one iteration against lm_step -> the largest pose and (relative) point differences"""
    dpo, dpt = lm_step(p["poses"], p["pose_fixed"], p["points"], p["e_point"], p["e_pose"], p["obs"], p["stereo"], p["inv_sigma2"], *p["cam"],
                       robust=p["robust"])
    po = poses.astype(np.float64) * np.where(poses[:, 3:4] < 0, -1.0, 1.0)
    d_pose = float(np.abs(po - dpo).max())
    d_pt = float((np.abs(points - dpt) / np.maximum(1.0, np.abs(dpt))).max())
    assert d_pose < tol and d_pt < tol, (d_pose, d_pt)
    return d_pose, d_pt

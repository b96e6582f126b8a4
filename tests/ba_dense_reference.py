"""One Levenberg-Marquardt step of local bundle adjustment, written from the definitions alone in numpy longdouble: an independent check
of the closed-form Jacobians, the per-edge blocks, the Schur complement and the back substitution that csrc/api_ba.cu and
oracle/ba_oracle.cpp share.  No Jacobian is written down here: every column is a central difference of the residual.

Definitions.  A key frame is T = (R, t) mapping world to camera, a point p is in the world, p_c = R p + t.
  residual of a mono edge    r = (u_obs, v_obs) - (fx x/z + cx, fy y/z + cy)                       with (x, y, z) = p_c
  residual of a stereo edge  r = (u_obs, v_obs, ur_obs) - (u, v, u - bf/z)
  (the stereo edge of the reference evaluates 1/z in float32; that rounding enters the residual here and not its derivatives, which
  cannot be differenced through a rounding step)
  robust cost                sum_k rho(s_k), s_k = info_k |r_k|^2, rho(s) = s for s <= d^2, else 2 d sqrt(s) - d^2 (Huber; d^2 = 5.991 for
                             mono, 7.815 for stereo), minimised by iteratively reweighted least squares: weight w_k = rho'(s_k) = 1 or
                             d / sqrt(s_k), no second-order term
  parametrisation            T <- exp(a) T for a = (omega, upsilon) in se(3), p <- p + b
                             exp(a) = (Rodrigues(omega), V upsilon), V = I + (1 - cos th)/th^2 [omega]x + (th - sin th)/th^3 [omega]x^2
  normal equations           H = sum_k w_k info_k J_k^T J_k, g = -sum_k w_k info_k J_k^T r_k, J_k = d r_k / d (a of its free key frame, b of
                             its point); the unknowns are the free key frames (6 each) then all points (3 each)
  step                       (H + lambda I) x = g, lambda = 1e-5 max |H_ii|, solved densely (Cholesky in longdouble)."""
import numpy as np

LD = np.longdouble
H_STEP = LD(1e-6)


def _skew(w):
    return np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]], LD)


def _rot(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]], LD)


def _exp(a):
    w, ups = a[:3], a[3:]
    th2 = w @ w
    W = _skew(w)
    if th2 < LD(1e-12):                                     # series: the differencing steps land here
        A, B, Cc = 1 - th2 / 6, LD(0.5) - th2 / 24, LD(1) / 6 - th2 / 120
    else:
        th = np.sqrt(th2)
        A, B, Cc = np.sin(th) / th, (1 - np.cos(th)) / th2, (th - np.sin(th)) / (th2 * th)
    I = np.eye(3, dtype=LD)
    return I + A * W + B * (W @ W), (I + B * W + Cc * (W @ W)) @ ups


def _project(R, t, p, cam, stereo, float_invz):
    fx, fy, cx, cy, bf = cam
    x, y, z = R @ p + t
    if not stereo:
        return np.array([fx * x / z + cx, fy * y / z + cy], LD)
    iz = LD(np.float32(1 / z)) if float_invz else 1 / z
    u = fx * x * iz + cx
    return np.array([u, fy * y * iz + cy, u - bf * iz], LD)


def _quat(R):
    """Rotation matrix -> (qx, qy, qz, qw) with qw >= 0 (largest-component branch)."""
    K = np.array([R[0, 0] + R[1, 1] + R[2, 2], R[0, 0] - R[1, 1] - R[2, 2], R[1, 1] - R[0, 0] - R[2, 2], R[2, 2] - R[0, 0] - R[1, 1]], LD)
    i = int(np.argmax(K))
    s = np.sqrt(1 + K[i]) * 2
    if i == 0:
        q = [(R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s, s / 4]
    elif i == 1:
        q = [s / 4, (R[0, 1] + R[1, 0]) / s, (R[0, 2] + R[2, 0]) / s, (R[2, 1] - R[1, 2]) / s]
    elif i == 2:
        q = [(R[0, 1] + R[1, 0]) / s, s / 4, (R[1, 2] + R[2, 1]) / s, (R[0, 2] - R[2, 0]) / s]
    else:
        q = [(R[0, 2] + R[2, 0]) / s, (R[1, 2] + R[2, 1]) / s, s / 4, (R[1, 0] - R[0, 1]) / s]
    q = np.array(q, LD)
    return q if q[3] >= 0 else -q


def _solve_spd(A, b):
    """Cholesky A = L L^T and the two substitutions, in the dtype of A."""
    n = len(b)
    L = A.copy()
    for k in range(n):
        assert L[k, k] > 0, "the damped normal equations are not positive definite"
        L[k, k] = np.sqrt(L[k, k])
        L[k + 1:, k] /= L[k, k]
        L[k + 1:, k + 1:] -= np.outer(L[k + 1:, k], L[k + 1:, k])
    y = b.copy()
    for k in range(n):
        y[k] /= L[k, k]
        y[k + 1:] -= L[k + 1:, k] * y[k]
    for k in range(n - 1, -1, -1):
        y[k] /= L[k, k]
        y[:k] -= L[k, :k] * y[k]
    return y


def lm_step(poses, pose_fixed, points, e_point, e_pose, obs, stereo, inv_sigma2, fx, fy, cx, cy, bf, iterations=1):
    """The estimates after the first LM trial, taken as accepted -> (poses[n, 7] with qw >= 0, points[m, 3]) in longdouble; fixed key
    frames are returned as given."""
    assert iterations == 1
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
        d2 = LD(7.815) if st else LD(5.991)
        w = LD(1) if s <= d2 else np.sqrt(d2 / s)
        J = np.zeros((d, 9), LD)                            # columns: omega, upsilon of the key frame, then the point
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
        Jk = J[:, 9 - len(idx):]                            # a fixed key frame contributes no unknowns
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

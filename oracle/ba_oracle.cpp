// ORACLE (test infrastructure, NOT product code): CPU restatement of Optimizer::LocalBundleAdjustment's numerical core
// (src/Optimizer.cc:1116-1499: vertices :1210-1295, edges :1297-1404, optimize(10) :1410-1411, outlier test :1416-1461) with
// the vendored g2o pieces it executes:
//   Levenberg-Marquardt + Raul's stop test   Thirdparty/g2o/g2o/core/optimization_algorithm_levenberg.cpp:61-201
//   optimize() loop                          core/sparse_optimizer.cpp:354-419
//   Schur complement block solver            core/block_solver.hpp:354-486 (Hschur = Hpp - sum_l Hpl Hll^-1 Hlp), buildSystem :501-560
//   binary-edge normal equations             core/base_binary_edge.hpp (no second-order robust term), Huber robust_kernel_impl.cpp:65-91
//   mono edge                                src/OptimizableTypes.cpp:139-160 (linearizeOplus), include/OptimizableTypes.h (computeError,
//                                            isDepthPositive), Pinhole::project / projectJac (src/CameraModels/Pinhole.cpp)
//   stereo edge                              types/types_six_dof_expmap.cpp:190-274 (float invz in cam_project)
//   vertex updates                           VertexSE3Expmap::oplusImpl (exp(delta) * T), VertexSBAPointXYZ::oplusImpl (+=)
// The graph is passed flat (what the C-ABI shim gathers): poses (fixed flag), points, edges (point, pose, obs, stereo flag,
// invSigma2).  The sparse Cholesky of the reduced system (LinearSolverEigen) is a dense LDL^T here: same solution up to
// rounding.  PARITY UNPINNED: g2o / Eigen cannot be built here; validated by convergence to ground truth and invariants.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>

namespace {

#include "g2o_se3.inc"

struct Cam { float fx, fy, cx, cy, bf; };

struct BAEdge { int point, pose; double obs[3]; double info; bool stereo; double err[3]; };

// What one call did (orc_local_bundle_adjustment_trace): every LM trial and iteration, how the run ended, and how close each discrete
// decision came to going the other way.  Margins are relative: for the accept / reject test the smaller of |rho| (already a ratio) and
// |chi2 - trial chi2| / chi2 (near convergence rho is a ratio of two rounding-sized numbers and says nothing about its own sign),
// |(ini - cur) * 1e3 - ini| / |ini| for the stop test, |e2 - delta^2| / delta^2 for the Huber switch, and per edge of the erase test
// min(|chi2 - threshold| / threshold, |z| / |p_camera|).  Decisions that do not depend on rounding (a failed solve, a non-finite
// value, 0 against 0) are not counted.  The per-trial / per-iteration / per-edge arrays belong to the caller (capacities cap_*).
struct BATrace {
    int cap_trials, cap_iters;
    double* trial_lambda; double* trial_rho; uint8_t* trial_accepted; uint8_t* trial_ok;
    int* iter_qmax; uint8_t* iter_bad; double* iter_margin;     // per iteration: trials run; of those that reached the stop test, its decision and margin
    double* edge_margin;                                        // n_edges: margin of each edge's erase test
    int n_trials, n_iters;
    int max_reject_run;                                         // most consecutive rejected trials in one iteration
    int term_qmax, term_nbad, term_rho0;                        // how the run ended (none set: the iteration limit)
    int solver_failures, ended_on_rejected_trial;
    double min_rho_margin, min_stop_margin, min_huber_margin, min_flag_margin, min_margin;
};

inline void margin(double& m, double dist, double scale) {
    if (std::isfinite(dist) && std::isfinite(scale) && scale != 0) m = std::min(m, std::fabs(dist) / std::fabs(scale));
}

struct BA {
    Cam cam;
    std::vector<SE3> poses; std::vector<uint8_t> fixed; std::vector<int> pose_slot;     // slot in the reduced system or -1
    std::vector<double> pts;                                                            // 3 per point
    std::vector<BAEdge> edges;
    int n_opt = 0;
    // system
    std::vector<double> Hpp, bp;       // n_opt x 36, n_opt x 6
    std::vector<double> Hll, bl;       // n_pts x 9, n_pts x 3
    std::vector<double> Hpl;           // per edge 18 (6 x 3), valid when the pose is not fixed
    std::vector<double> x;             // solution: poses then points
    double lambda = 0, ni = 2; int n_bad = 0;
    BATrace* tr = nullptr;
    const double delta_mono = (double)(float)std::sqrt(5.991), delta_stereo = (double)(float)std::sqrt(7.815);

    void edge_error(BAEdge& e) const {
        double p[3];
        se3_map(poses[e.pose], &pts[3 * e.point], p);
        if (e.stereo) {
            const double fx = cam.fx, fy = cam.fy, cx = cam.cx, cy = cam.cy;
            const float invz = 1.0f / p[2];
            const double u = p[0] * invz * fx + cx, v = p[1] * invz * fy + cy;
            e.err[0] = e.obs[0] - u; e.err[1] = e.obs[1] - v; e.err[2] = e.obs[2] - (u - cam.bf * invz);
        } else {
            e.err[0] = e.obs[0] - ((double)cam.fx * p[0] / p[2] + (double)cam.cx);       // Pinhole::project(Vector3d)
            e.err[1] = e.obs[1] - ((double)cam.fy * p[1] / p[2] + (double)cam.cy);
            e.err[2] = 0;
        }
    }
    static void huber(double e2, double delta, float dsqr, double rho[2]) {
        if (e2 <= dsqr) { rho[0] = e2; rho[1] = 1.; }
        else { const double sq = std::sqrt(e2); rho[0] = 2 * sq * delta - dsqr; rho[1] = delta / sq; }
    }
    double chi2(const BAEdge& e) const { return e.info * (e.err[0] * e.err[0] + e.err[1] * e.err[1] + e.err[2] * e.err[2]); }
    double active_robust_chi2() {
        double s = 0;
        for (auto& e : edges) {
            double rho[2];
            const double d = e.stereo ? delta_stereo : delta_mono;
            huber(chi2(e), d, (float)(d * d), rho);
            if (tr) margin(tr->min_huber_margin, chi2(e) - (double)(float)(d * d), (double)(float)(d * d));
            s += rho[0];
        }
        return s;
    }
    void compute_errors() { for (auto& e : edges) edge_error(e); }

    void jacobians(const BAEdge& e, double Jl[3][3], double Jp[3][6]) const {
        const SE3& T = poses[e.pose];
        double p[3];
        se3_map(T, &pts[3 * e.point], p);
        const double x = p[0], y = p[1], z = p[2], z2 = z * z;
        double R[3][3];                                       // Quaterniond::toRotationMatrix
        {
            const Quat& q = T.r;
            const double tx = 2 * q.x, ty = 2 * q.y, tz = 2 * q.z, twx = tx * q.w, twy = ty * q.w, twz = tz * q.w,
                         txx = tx * q.x, txy = ty * q.x, txz = tz * q.x, tyy = ty * q.y, tyz = tz * q.y, tzz = tz * q.z;
            R[0][0] = 1 - (tyy + tzz); R[0][1] = txy - twz; R[0][2] = txz + twy;
            R[1][0] = txy + twz; R[1][1] = 1 - (txx + tzz); R[1][2] = tyz - twx;
            R[2][0] = txz - twy; R[2][1] = tyz + twx; R[2][2] = 1 - (txx + tyy);
        }
        const double fx = cam.fx, fy = cam.fy, bf = cam.bf;
        if (e.stereo) {
            for (int c = 0; c < 3; ++c) {
                Jl[0][c] = -fx * R[0][c] / z + fx * x * R[2][c] / z2;
                Jl[1][c] = -fy * R[1][c] / z + fy * y * R[2][c] / z2;
                Jl[2][c] = Jl[0][c] - bf * R[2][c] / z2;
            }
            Jp[0][0] = x * y / z2 * fx; Jp[0][1] = -(1 + (x * x / z2)) * fx; Jp[0][2] = y / z * fx; Jp[0][3] = -1. / z * fx; Jp[0][4] = 0; Jp[0][5] = x / z2 * fx;
            Jp[1][0] = (1 + y * y / z2) * fy; Jp[1][1] = -x * y / z2 * fy; Jp[1][2] = -x / z * fy; Jp[1][3] = 0; Jp[1][4] = -1. / z * fy; Jp[1][5] = y / z2 * fy;
            Jp[2][0] = Jp[0][0] - bf * y / z2; Jp[2][1] = Jp[0][1] + bf * x / z2; Jp[2][2] = Jp[0][2]; Jp[2][3] = Jp[0][3]; Jp[2][4] = 0; Jp[2][5] = Jp[0][5] - bf / z2;
        } else {
            const double pj[2][3] = {{-(fx / z), -0.0, -(-fx * x / z2)}, {-0.0, -(fy / z), -(-fy * y / z2)}};     // -projectJac
            for (int r = 0; r < 2; ++r)
                for (int c = 0; c < 3; ++c) Jl[r][c] = pj[r][0] * R[0][c] + pj[r][1] * R[1][c] + pj[r][2] * R[2][c];
            const double D[3][6] = {{0, z, -y, 1, 0, 0}, {-z, 0, x, 0, 1, 0}, {y, -x, 0, 0, 0, 1}};
            for (int r = 0; r < 2; ++r)
                for (int c = 0; c < 6; ++c) Jp[r][c] = pj[r][0] * D[0][c] + pj[r][1] * D[1][c] + pj[r][2] * D[2][c];
            for (int c = 0; c < 3; ++c) Jl[2][c] = 0;
            for (int c = 0; c < 6; ++c) Jp[2][c] = 0;
        }
    }

    void build_system() {
        const int np = (int)pts.size() / 3;
        Hpp.assign((size_t)n_opt * 36, 0); bp.assign((size_t)n_opt * 6, 0);
        Hll.assign((size_t)np * 9, 0); bl.assign((size_t)np * 3, 0);
        Hpl.assign(edges.size() * 18, 0);
        for (size_t k = 0; k < edges.size(); ++k) {
            const BAEdge& e = edges[k];
            double Jl[3][3], Jp[3][6], rho[2];
            jacobians(e, Jl, Jp);
            const double d = e.stereo ? delta_stereo : delta_mono;
            huber(chi2(e), d, (float)(d * d), rho);
            const double w = rho[1] * e.info;
            double we[3] = {-rho[1] * e.info * e.err[0], -rho[1] * e.info * e.err[1], -rho[1] * e.info * e.err[2]};   // omega_r = -Omega e, robustified
            double* hl = &Hll[9 * (size_t)e.point]; double* b_l = &bl[3 * (size_t)e.point];
            for (int i = 0; i < 3; ++i) {
                for (int j = 0; j < 3; ++j) { double s = 0; for (int r = 0; r < 3; ++r) s += Jl[r][i] * w * Jl[r][j]; hl[3 * i + j] += s; }
                double s = 0; for (int r = 0; r < 3; ++r) s += Jl[r][i] * we[r];
                b_l[i] += s;
            }
            const int slot = pose_slot[e.pose];
            if (slot >= 0) {
                double* hp = &Hpp[36 * (size_t)slot]; double* b_p = &bp[6 * (size_t)slot]; double* hpl = &Hpl[18 * k];
                for (int i = 0; i < 6; ++i) {
                    for (int j = 0; j < 6; ++j) { double s = 0; for (int r = 0; r < 3; ++r) s += Jp[r][i] * w * Jp[r][j]; hp[6 * i + j] += s; }
                    for (int j = 0; j < 3; ++j) { double s = 0; for (int r = 0; r < 3; ++r) s += Jp[r][i] * w * Jl[r][j]; hpl[3 * i + j] = s; }
                    double s = 0; for (int r = 0; r < 3; ++r) s += Jp[r][i] * we[r];
                    b_p[i] += s;
                }
            }
        }
    }

    static bool inv3(const double* m, double* o) {
        const double a = m[0], b = m[1], c = m[2], d = m[3], e = m[4], f = m[5], g = m[6], h = m[7], i = m[8];
        const double det = a * (e * i - f * h) - b * (d * i - f * g) + c * (d * h - e * g);
        const double id = 1.0 / det;
        o[0] = (e * i - f * h) * id; o[1] = (c * h - b * i) * id; o[2] = (b * f - c * e) * id;
        o[3] = (f * g - d * i) * id; o[4] = (a * i - c * g) * id; o[5] = (c * d - a * f) * id;
        o[6] = (d * h - e * g) * id; o[7] = (b * g - a * h) * id; o[8] = (a * e - b * d) * id;
        return std::isfinite(id);
    }

    // (H + lambda I) x = b through the Schur complement; dense LDL^T of the reduced pose system
    bool solve(double lam) {
        const int np = (int)pts.size() / 3, n = 6 * n_opt;
        std::vector<double> S((size_t)n * n, 0.0), bs(n, 0.0), Dinv((size_t)np * 9), coef(n, 0.0);
        for (int s = 0; s < n_opt; ++s)
            for (int i = 0; i < 6; ++i) {
                for (int j = 0; j < 6; ++j) S[(size_t)(6 * s + i) * n + 6 * s + j] = Hpp[36 * (size_t)s + 6 * i + j];
                S[(size_t)(6 * s + i) * n + 6 * s + i] += lam;
            }
        std::vector<std::vector<int>> by_point(np);
        for (size_t k = 0; k < edges.size(); ++k) if (pose_slot[edges[k].pose] >= 0) by_point[edges[k].point].push_back((int)k);
        for (int l = 0; l < np; ++l) {
            double D[9];
            for (int i = 0; i < 9; ++i) D[i] = Hll[9 * (size_t)l + i];
            D[0] += lam; D[4] += lam; D[8] += lam;
            inv3(D, &Dinv[9 * (size_t)l]);
            const double* di = &Dinv[9 * (size_t)l];
            double db[3];
            for (int i = 0; i < 3; ++i) db[i] = di[3 * i] * bl[3 * l] + di[3 * i + 1] * bl[3 * l + 1] + di[3 * i + 2] * bl[3 * l + 2];
            for (int k1 : by_point[l]) {
                const int s1 = pose_slot[edges[k1].pose];
                const double* B1 = &Hpl[18 * (size_t)k1];
                double BD[18];
                for (int i = 0; i < 6; ++i)
                    for (int j = 0; j < 3; ++j) BD[3 * i + j] = B1[3 * i] * di[j] + B1[3 * i + 1] * di[3 + j] + B1[3 * i + 2] * di[6 + j];
                for (int i = 0; i < 6; ++i) coef[6 * s1 + i] += B1[3 * i] * db[0] + B1[3 * i + 1] * db[1] + B1[3 * i + 2] * db[2];
                for (int k2 : by_point[l]) {
                    const int s2 = pose_slot[edges[k2].pose];
                    const double* B2 = &Hpl[18 * (size_t)k2];
                    for (int i = 0; i < 6; ++i)
                        for (int j = 0; j < 6; ++j)
                            S[(size_t)(6 * s1 + i) * n + 6 * s2 + j] -= BD[3 * i] * B2[3 * j] + BD[3 * i + 1] * B2[3 * j + 1] + BD[3 * i + 2] * B2[3 * j + 2];
                }
            }
        }
        for (int i = 0; i < n; ++i) bs[i] = bp[i] - coef[i];
        // LDL^T without pivoting (SPD), fails on a non-positive pivot like a Cholesky does
        std::vector<double> d(n);
        for (int k = 0; k < n; ++k) {
            double dk = S[(size_t)k * n + k];
            for (int m = 0; m < k; ++m) dk -= S[(size_t)k * n + m] * S[(size_t)k * n + m] * d[m];
            if (!(dk > 0) || !std::isfinite(dk)) return false;
            d[k] = dk;
            for (int i = k + 1; i < n; ++i) {
                double v = S[(size_t)i * n + k];
                for (int m = 0; m < k; ++m) v -= S[(size_t)i * n + m] * S[(size_t)k * n + m] * d[m];
                S[(size_t)i * n + k] = v / dk;
            }
        }
        std::vector<double> y(bs);
        for (int i = 0; i < n; ++i) for (int m = 0; m < i; ++m) y[i] -= S[(size_t)i * n + m] * y[m];
        for (int i = 0; i < n; ++i) y[i] /= d[i];
        for (int i = n - 1; i >= 0; --i) for (int m = i + 1; m < n; ++m) y[i] -= S[(size_t)m * n + i] * y[m];
        x.assign((size_t)n + 3 * np, 0.0);
        for (int i = 0; i < n; ++i) x[i] = y[i];
        // landmarks: xl = Dinv (bl - Hpl^T xp)
        std::vector<double> cl(bl);
        for (size_t k = 0; k < edges.size(); ++k) {
            const int s = pose_slot[edges[k].pose];
            if (s < 0) continue;
            const double* B = &Hpl[18 * k];
            for (int j = 0; j < 3; ++j) {
                double v = 0;
                for (int i = 0; i < 6; ++i) v += B[3 * i + j] * x[6 * s + i];
                cl[3 * (size_t)edges[k].point + j] -= v;
            }
        }
        for (int l = 0; l < np; ++l) {
            const double* di = &Dinv[9 * (size_t)l];
            for (int i = 0; i < 3; ++i) x[n + 3 * l + i] = di[3 * i] * cl[3 * l] + di[3 * i + 1] * cl[3 * l + 1] + di[3 * i + 2] * cl[3 * l + 2];
        }
        return true;
    }

    void apply_update() {
        const int np = (int)pts.size() / 3, n = 6 * n_opt;
        for (size_t p = 0; p < poses.size(); ++p) {
            const int s = pose_slot[p];
            if (s < 0) continue;
            poses[p] = se3_mul(se3_exp(&x[6 * s]), poses[p]);
        }
        for (int l = 0; l < np; ++l) for (int i = 0; i < 3; ++i) pts[3 * l + i] += x[n + 3 * l + i];
    }

    // returns 0 OK, 1 Terminate
    int lm_iteration(int iteration) {
        compute_errors();
        double current = active_robust_chi2(), temp = current;
        const double ini = current;
        build_system();
        const int np = (int)pts.size() / 3, n = 6 * n_opt;
        if (iteration == 0) {
            double mx = 0;
            for (int s = 0; s < n_opt; ++s) for (int j = 0; j < 6; ++j) mx = std::max(std::fabs(Hpp[36 * (size_t)s + 7 * j]), mx);
            for (int l = 0; l < np; ++l) for (int j = 0; j < 3; ++j) mx = std::max(std::fabs(Hll[9 * (size_t)l + 4 * j]), mx);
            lambda = 1e-5 * mx; ni = 2; n_bad = 0;
        }
        double rho = 0; int qmax = 0, reject_run = 0;
        do {
            const std::vector<SE3> backup_poses = poses; const std::vector<double> backup_pts = pts;      // push()
            const bool ok2 = solve(lambda);
            if (ok2) apply_update(); else x.assign((size_t)n + 3 * np, 0.0);
            compute_errors();
            temp = active_robust_chi2();
            if (!ok2) temp = std::numeric_limits<double>::max();
            rho = current - temp;
            double scale = 0;
            for (int j = 0; j < n; ++j) scale += x[j] * (lambda * x[j] + bp[j]);
            for (int j = 0; j < 3 * np; ++j) scale += x[n + j] * (lambda * x[n + j] + bl[j]);
            scale += 1e-3;
            rho /= scale;
            if (tr) {
                const bool accepted = rho > 0 && std::isfinite(temp);
                if (tr->n_trials < tr->cap_trials) {
                    tr->trial_lambda[tr->n_trials] = lambda; tr->trial_rho[tr->n_trials] = rho;
                    tr->trial_accepted[tr->n_trials] = accepted; tr->trial_ok[tr->n_trials] = ok2;
                }
                ++tr->n_trials;
                if (!ok2) ++tr->solver_failures;
                if (ok2 && !(current == 0 && temp == 0) && std::isfinite(rho)) {
                    tr->min_rho_margin = std::min(tr->min_rho_margin, std::fabs(rho));
                    margin(tr->min_rho_margin, current - temp, std::max(current, temp));
                }
                tr->ended_on_rejected_trial = !accepted;
                reject_run = accepted ? 0 : reject_run + 1;
                tr->max_reject_run = std::max(tr->max_reject_run, reject_run);
            }
            if (rho > 0 && std::isfinite(temp)) {
                double alpha = 1. - std::pow(2 * rho - 1, 3);
                alpha = std::min(alpha, 2. / 3.);
                lambda *= std::max(1. / 3., alpha); ni = 2; current = temp;
            } else {
                lambda *= ni; ni *= 2; poses = backup_poses; pts = backup_pts;                        // pop()
            }
            ++qmax;
        } while (rho < 0 && qmax < 10);
        if (tr) {
            const int i = tr->n_iters++;
            const bool stop = qmax == 10 || rho == 0;
            if (qmax == 10) tr->term_qmax = 1; else if (rho == 0) tr->term_rho0 = 1;
            if (i < tr->cap_iters) {
                tr->iter_qmax[i] = qmax; tr->iter_bad[i] = !stop && (ini - current) * 1e3 < ini;
                tr->iter_margin[i] = std::numeric_limits<double>::infinity();
                if (!stop && ini != 0) margin(tr->iter_margin[i], (ini - current) * 1e3 - ini, ini);
            }
            if (!stop && ini != 0) margin(tr->min_stop_margin, (ini - current) * 1e3 - ini, ini);
            if (!stop && (ini - current) * 1e3 < ini && n_bad + 1 >= 3) tr->term_nbad = 1;
        }
        if (qmax == 10 || rho == 0) return 1;
        if ((ini - current) * 1e3 < ini) ++n_bad; else n_bad = 0;
        if (n_bad >= 3) return 1;
        return 0;
    }
};

// poses: n_poses x 7 floats (qx qy qz qw tx ty tz, Tcw); pose_fixed[n_poses]; points: n_points x 3 floats;
// edges: e_point, e_pose, obs (n_edges x 3 floats: u, v, ur), stereo flags, inv_sigma2.  Outputs: optimised poses / points (float,
// fixed poses unchanged) and per edge the reference's erase test (chi2 > 5.991 / 7.815 with the errors of the LAST evaluated
// trial, or non-positive depth at the final estimates).  Returns the number of LM iterations run.
int local_bundle_adjustment(int n_poses, const float* poses, const uint8_t* pose_fixed, int n_points, const float* points, int n_edges,
                            const int32_t* e_point, const int32_t* e_pose, const float* obs, const uint8_t* stereo,
                            const float* inv_sigma2, float fx, float fy, float cx, float cy, float bf, int iterations,
                            float* poses_out, float* points_out, uint8_t* edge_erase, double* final_chi2, BATrace* tr) {
    BA ba;
    ba.tr = tr;
    ba.cam = Cam{fx, fy, cx, cy, bf};
    ba.poses.resize(n_poses); ba.fixed.assign(pose_fixed, pose_fixed + n_poses); ba.pose_slot.resize(n_poses);
    for (int p = 0; p < n_poses; ++p) {
        SE3 T; T.r = Quat{poses[7 * p], poses[7 * p + 1], poses[7 * p + 2], poses[7 * p + 3]};
        T.t[0] = poses[7 * p + 4]; T.t[1] = poses[7 * p + 5]; T.t[2] = poses[7 * p + 6];
        normalize_rotation(T);                               // SE3Quat(q, t) constructor
        ba.poses[p] = T;
        ba.pose_slot[p] = pose_fixed[p] ? -1 : ba.n_opt++;
    }
    ba.pts.assign(points, points + 3 * (size_t)n_points);
    ba.edges.resize(n_edges);
    for (int k = 0; k < n_edges; ++k) {
        BAEdge& e = ba.edges[k];
        e.point = e_point[k]; e.pose = e_pose[k]; e.stereo = stereo[k] != 0; e.info = inv_sigma2[k];
        e.obs[0] = obs[3 * k]; e.obs[1] = obs[3 * k + 1]; e.obs[2] = obs[3 * k + 2];
        e.err[0] = e.err[1] = e.err[2] = 0;
    }
    int it = 0;
    if (n_edges > 0 && (ba.n_opt > 0 || n_points > 0))
        for (; it < iterations; ++it) { if (ba.lm_iteration(it) != 0) { ++it; break; } }
    for (int p = 0; p < n_poses; ++p) {
        const SE3& T = ba.poses[p];
        if (pose_fixed[p]) { for (int i = 0; i < 7; ++i) poses_out[7 * p + i] = poses[7 * p + i]; continue; }
        poses_out[7 * p] = (float)T.r.x; poses_out[7 * p + 1] = (float)T.r.y; poses_out[7 * p + 2] = (float)T.r.z; poses_out[7 * p + 3] = (float)T.r.w;
        poses_out[7 * p + 4] = (float)T.t[0]; poses_out[7 * p + 5] = (float)T.t[1]; poses_out[7 * p + 6] = (float)T.t[2];
    }
    for (size_t i = 0; i < ba.pts.size(); ++i) points_out[i] = (float)ba.pts[i];
    for (int k = 0; k < n_edges; ++k) {
        const BAEdge& e = ba.edges[k];
        double p[3];
        se3_map(ba.poses[e.pose], &ba.pts[3 * (size_t)e.point], p);
        edge_erase[k] = (ba.chi2(e) > (e.stereo ? 7.815 : 5.991) || !(p[2] > 0.0)) ? 1 : 0;
        if (tr) {
            double m = std::numeric_limits<double>::infinity();
            margin(m, ba.chi2(e) - (e.stereo ? 7.815 : 5.991), e.stereo ? 7.815 : 5.991);
            margin(m, p[2], std::sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2]));
            tr->edge_margin[k] = m;
            tr->min_flag_margin = std::min(tr->min_flag_margin, m);
        }
    }
    if (tr) tr->min_margin = std::min(std::min(tr->min_rho_margin, tr->min_stop_margin), std::min(tr->min_huber_margin, tr->min_flag_margin));
    ba.tr = nullptr;
    if (final_chi2) { *final_chi2 = ba.active_robust_chi2(); }
    return it;
}

}  // namespace

extern "C" {

int orc_local_bundle_adjustment(int n_poses, const float* poses, const uint8_t* pose_fixed, int n_points, const float* points, int n_edges,
                                const int32_t* e_point, const int32_t* e_pose, const float* obs, const uint8_t* stereo,
                                const float* inv_sigma2, float fx, float fy, float cx, float cy, float bf, int iterations,
                                float* poses_out, float* points_out, uint8_t* edge_erase, double* final_chi2) {
    return local_bundle_adjustment(n_poses, poses, pose_fixed, n_points, points, n_edges, e_point, e_pose, obs, stereo, inv_sigma2, fx, fy, cx, cy, bf, iterations,
                                   poses_out, points_out, edge_erase, final_chi2, nullptr);
}

// orc_local_bundle_adjustment with the same arithmetic and outputs, plus what the call did (BATrace above); the caller sets the
// capacities and array pointers of *tr
int orc_local_bundle_adjustment_trace(int n_poses, const float* poses, const uint8_t* pose_fixed, int n_points, const float* points, int n_edges,
                                      const int32_t* e_point, const int32_t* e_pose, const float* obs, const uint8_t* stereo,
                                      const float* inv_sigma2, float fx, float fy, float cx, float cy, float bf, int iterations,
                                      float* poses_out, float* points_out, uint8_t* edge_erase, double* final_chi2, BATrace* tr) {
    tr->n_trials = tr->n_iters = tr->max_reject_run = tr->term_qmax = tr->term_nbad = tr->term_rho0 = tr->solver_failures = tr->ended_on_rejected_trial = 0;
    tr->min_rho_margin = tr->min_stop_margin = tr->min_huber_margin = tr->min_flag_margin = tr->min_margin = std::numeric_limits<double>::infinity();
    return local_bundle_adjustment(n_poses, poses, pose_fixed, n_points, points, n_edges, e_point, e_pose, obs, stereo, inv_sigma2, fx, fy, cx, cy, bf, iterations,
                                   poses_out, points_out, edge_erase, final_chi2, tr);
}

}  // extern "C"

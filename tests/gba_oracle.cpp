// ORACLE (test infrastructure, NOT product code): CPU restatement of Optimizer::BundleAdjustment's numerical core (src/Optimizer.cc:60;
// GlobalBundleAdjustemnt :52 calls it) over the flat graph of rgbl_global_bundle_adjustment.  It is oracle/ba_oracle.cpp's local-BA
// restatement (compiled into this library unchanged: its Jacobians, Schur solve, updates and trace) with what BundleAdjustment does
// differently:
//   robust kernel   Huber only when bRobust, deltas sqrt(5.99) mono and sqrt(7.815) stereo (local BA: sqrt(5.991) mono, always on);
//                   without it g2o's robustify is skipped: rho(e2) = e2, weight 1
//   stop flag       pbStopFlag is g2o's force-stop flag: read before every iteration (core/sparse_optimizer.cpp optimize()) and after
//                   every trial (the `while (rho < 0 && qmax < 10 && !terminate())` of optimization_algorithm_levenberg.cpp)
//   no outlier pass and no second optimisation; points without edges stay out of the graph (vbNotIncludedMP) and come back unchanged
// The reading of the reference used is that of its optimize(nIterations) after initializeOptimization(), as in local BA.
#include "ba_oracle.cpp"

namespace {

struct GBA : BA {
    bool robust = false;
    double dm = 0, ds = 0;                     // Huber deltas (float, as g2o's setDelta stores them)
    const volatile uint8_t* stop = nullptr;

    bool stopped() const { return stop && *stop != 0; }
    void rho_of(double e2, bool stereo, double rho[2]) const {
        if (!robust) { rho[0] = e2; rho[1] = 1.; return; }
        const double d = stereo ? ds : dm;
        huber(e2, d, (float)(d * d), rho);
    }
    double active_robust_chi2() {
        double s = 0;
        for (auto& e : edges) {
            double rho[2];
            rho_of(chi2(e), e.stereo, rho);
            if (tr && robust) { const double d = e.stereo ? ds : dm; margin(tr->min_huber_margin, chi2(e) - (double)(float)(d * d), (double)(float)(d * d)); }
            s += rho[0];
        }
        return s;
    }
    // BA::build_system with rho_of for the fixed Huber kernel
    void build_system() {
        const int np = (int)pts.size() / 3;
        Hpp.assign((size_t)n_opt * 36, 0); bp.assign((size_t)n_opt * 6, 0);
        Hll.assign((size_t)np * 9, 0); bl.assign((size_t)np * 3, 0);
        Hpl.assign(edges.size() * 18, 0);
        for (size_t k = 0; k < edges.size(); ++k) {
            const BAEdge& e = edges[k];
            double Jl[3][3], Jp[3][6], rho[2];
            jacobians(e, Jl, Jp);
            rho_of(chi2(e), e.stereo, rho);
            const double w = rho[1] * e.info;
            double we[3] = {-rho[1] * e.info * e.err[0], -rho[1] * e.info * e.err[1], -rho[1] * e.info * e.err[2]};
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
    // BA::lm_iteration with the stop flag in the trial loop; returns 0 OK, 1 Terminate
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
            const std::vector<SE3> backup_poses = poses; const std::vector<double> backup_pts = pts;
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
                lambda *= ni; ni *= 2; poses = backup_poses; pts = backup_pts;
            }
            ++qmax;
        } while (rho < 0 && qmax < 10 && !stopped());
        if (tr) {
            const int i = tr->n_iters++;
            const bool stop_now = qmax == 10 || rho == 0;
            if (qmax == 10) tr->term_qmax = 1; else if (rho == 0) tr->term_rho0 = 1;
            if (i < tr->cap_iters) {
                tr->iter_qmax[i] = qmax; tr->iter_bad[i] = !stop_now && (ini - current) * 1e3 < ini;
                tr->iter_margin[i] = std::numeric_limits<double>::infinity();
                if (!stop_now && ini != 0) margin(tr->iter_margin[i], (ini - current) * 1e3 - ini, ini);
            }
            if (!stop_now && ini != 0) margin(tr->min_stop_margin, (ini - current) * 1e3 - ini, ini);
            if (!stop_now && (ini - current) * 1e3 < ini && n_bad + 1 >= 3) tr->term_nbad = 1;
        }
        if (qmax == 10 || rho == 0) return 1;
        if ((ini - current) * 1e3 < ini) ++n_bad; else n_bad = 0;
        if (n_bad >= 3) return 1;
        return 0;
    }
};

int global_bundle_adjustment(int n_poses, const float* poses, const uint8_t* pose_fixed, int n_points, const float* points, int n_edges,
                             const int32_t* e_point, const int32_t* e_pose, const float* obs, const uint8_t* stereo, const float* inv_sigma2,
                             float fx, float fy, float cx, float cy, float bf, int iterations, int robust, const volatile uint8_t* stop,
                             float* poses_out, float* points_out, double* final_chi2, BATrace* tr) {
    GBA ba;
    ba.tr = tr;
    ba.robust = robust != 0;
    ba.dm = (double)(float)std::sqrt(5.99); ba.ds = (double)(float)std::sqrt(7.815);
    ba.stop = stop;
    ba.cam = Cam{fx, fy, cx, cy, bf};
    ba.poses.resize(n_poses); ba.fixed.assign(pose_fixed, pose_fixed + n_poses); ba.pose_slot.resize(n_poses);
    for (int p = 0; p < n_poses; ++p) {
        SE3 T; T.r = Quat{poses[7 * p], poses[7 * p + 1], poses[7 * p + 2], poses[7 * p + 3]};
        T.t[0] = poses[7 * p + 4]; T.t[1] = poses[7 * p + 5]; T.t[2] = poses[7 * p + 6];
        normalize_rotation(T);
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
    if (n_edges > 0)
        for (; it < iterations && !ba.stopped(); ++it) { if (ba.lm_iteration(it) != 0) { ++it; break; } }
    for (int p = 0; p < n_poses; ++p) {
        const SE3& T = ba.poses[p];
        if (pose_fixed[p]) { for (int i = 0; i < 7; ++i) poses_out[7 * p + i] = poses[7 * p + i]; continue; }
        poses_out[7 * p] = (float)T.r.x; poses_out[7 * p + 1] = (float)T.r.y; poses_out[7 * p + 2] = (float)T.r.z; poses_out[7 * p + 3] = (float)T.r.w;
        poses_out[7 * p + 4] = (float)T.t[0]; poses_out[7 * p + 5] = (float)T.t[1]; poses_out[7 * p + 6] = (float)T.t[2];
    }
    for (size_t i = 0; i < ba.pts.size(); ++i) points_out[i] = (float)ba.pts[i];
    if (tr) {
        tr->min_flag_margin = std::numeric_limits<double>::infinity();          // no erase test in BundleAdjustment
        tr->min_margin = std::min(std::min(tr->min_rho_margin, tr->min_stop_margin), tr->min_huber_margin);
    }
    ba.tr = nullptr;
    if (final_chi2) { ba.compute_errors(); *final_chi2 = ba.active_robust_chi2(); }
    return it;
}

}  // namespace

extern "C" {

// Optimizer::BundleAdjustment on the flat graph -> LM iterations run; optimised poses (fixed ones as given) and points.  stop: nullable,
// read before every iteration and after every trial.  tr: nullable, BATrace of oracle/ba_oracle.cpp (edge_margin is not written)
int orc_global_bundle_adjustment_trace(int n_poses, const float* poses, const uint8_t* pose_fixed, int n_points, const float* points, int n_edges,
                                       const int32_t* e_point, const int32_t* e_pose, const float* obs, const uint8_t* stereo,
                                       const float* inv_sigma2, float fx, float fy, float cx, float cy, float bf, int iterations, int robust,
                                       const uint8_t* stop, float* poses_out, float* points_out, double* final_chi2, BATrace* tr) {
    if (tr) {
        tr->n_trials = tr->n_iters = tr->max_reject_run = tr->term_qmax = tr->term_nbad = tr->term_rho0 = tr->solver_failures = tr->ended_on_rejected_trial = 0;
        tr->min_rho_margin = tr->min_stop_margin = tr->min_huber_margin = tr->min_flag_margin = tr->min_margin = std::numeric_limits<double>::infinity();
    }
    return global_bundle_adjustment(n_poses, poses, pose_fixed, n_points, points, n_edges, e_point, e_pose, obs, stereo, inv_sigma2, fx, fy, cx, cy, bf,
                                    iterations, robust, stop, poses_out, points_out, final_chi2, tr);
}

int orc_global_bundle_adjustment(int n_poses, const float* poses, const uint8_t* pose_fixed, int n_points, const float* points, int n_edges,
                                 const int32_t* e_point, const int32_t* e_pose, const float* obs, const uint8_t* stereo, const float* inv_sigma2,
                                 float fx, float fy, float cx, float cy, float bf, int iterations, int robust, const uint8_t* stop,
                                 float* poses_out, float* points_out, double* final_chi2) {
    return orc_global_bundle_adjustment_trace(n_poses, poses, pose_fixed, n_points, points, n_edges, e_point, e_pose, obs, stereo, inv_sigma2, fx, fy, cx,
                                              cy, bf, iterations, robust, stop, poses_out, points_out, final_chi2, nullptr);
}

}  // extern "C"

// ORACLE (test infrastructure, NOT product code): CPU restatement of Optimizer::PoseOptimization
// (src/Optimizer.cc:814-1114) with the vendored g2o pieces it executes:
//   Levenberg-Marquardt      Thirdparty/g2o/g2o/core/optimization_algorithm_levenberg.cpp:61-185
//   optimize() loop          core/sparse_optimizer.cpp:354-419, activeRobustChi2 :100-114
//   unary-edge normal eqs    core/base_unary_edge.hpp:43-72 (no second-order robust term, base_edge.h:96-102)
//   Huber kernel             core/robust_kernel_impl.cpp:65-91 (NOTE: dsqr is a *float* member, robust_kernel_impl.h:84)
//   SE3Quat map/exp/product  types/se3quat.h:104-110,214-254,280-285; VertexSE3Expmap::oplusImpl types_six_dof_expmap.h:73-76
//   stereo pose-only edge    types/types_six_dof_expmap.cpp:339-404 (float invz in cam_project), .h:218-222
//   mono pose-only edge      src/OptimizableTypes.cpp:49-63, include/OptimizableTypes.h:38-42, Pinhole.cpp:38-44,71-81
// Eigen (un-vendored) pieces are restated: Quaterniond * Vector3d, Quaterniond(Matrix3d), 6x6 LDLT solve.
// PINNED (round 2): tests/test_oracle_tracking_ref.py compares this file with the reference's own Optimizer::PoseOptimization body
// (src/Optimizer.cc:814-1114) running on the reference's g2o, both compiled unmodified over a stand-in Eigen (oracle/ref_tracking_driver.cpp):
// identical outlier flags and inlier counts, poses equal to 1e-6 on 8 problem families + degenerate sizes.
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <vector>

namespace {

#include "g2o_se3.inc"

struct Edge {
    double xw[3], obs[3];
    double info;         // invSigma2 (float in the Frame, widened)
    bool stereo;
    // state
    int level = 0;       // 0 active, 1 outlier
    bool robust = true;
    double err[3] = {0, 0, 0};
};

struct Cam { float fx, fy, cx, cy, bf; };

inline void edge_error(Edge& e, const SE3& T, const Cam& c) {
    double p[3];
    se3_map(T, e.xw, p);
    if (e.stereo) {
        const double fx = c.fx, fy = c.fy, cx = c.cx, cy = c.cy, bf = c.bf;      // edge members are double
        const float invz = 1.0f / p[2];                                          // types_six_dof_expmap.cpp:340
        const double u = p[0] * invz * fx + cx, v = p[1] * invz * fy + cy;
        e.err[0] = e.obs[0] - u; e.err[1] = e.obs[1] - v; e.err[2] = e.obs[2] - (u - bf * invz);
    } else {
        e.err[0] = e.obs[0] - (c.fx * p[0] / p[2] + c.cx);                       // Pinhole::project(Vector3d): float params widen
        e.err[1] = e.obs[1] - (c.fy * p[1] / p[2] + c.cy);
        e.err[2] = 0;
    }
}

inline double edge_chi2(const Edge& e) {
    const int d = e.stereo ? 3 : 2;
    double s = 0;
    for (int i = 0; i < d; ++i) s += e.err[i] * (e.info * e.err[i]);
    return s;
}

inline void huber(double e2, double delta, float dsqr, double rho[3]) {         // robust_kernel_impl.cpp:78-91
    if (e2 <= dsqr) { rho[0] = e2; rho[1] = 1.; rho[2] = 0.; }
    else {
        const double sq = std::sqrt(e2);
        rho[0] = 2 * sq * delta - dsqr;
        rho[1] = delta / sq;
        rho[2] = -0.5 * rho[1] / e2;
    }
}

inline void edge_jacobian(const Edge& e, const SE3& T, const Cam& c, double J[3][6]) {
    double p[3];
    se3_map(T, e.xw, p);
    const double x = p[0], y = p[1];
    if (e.stereo) {
        const double fx = c.fx, fy = c.fy, bf = c.bf;
        const double invz = 1.0 / p[2], invz_2 = invz * invz;
        J[0][0] = x * y * invz_2 * fx;  J[0][1] = -(1 + (x * x * invz_2)) * fx; J[0][2] = y * invz * fx;
        J[0][3] = -invz * fx;           J[0][4] = 0;                           J[0][5] = x * invz_2 * fx;
        J[1][0] = (1 + y * y * invz_2) * fy; J[1][1] = -x * y * invz_2 * fy;   J[1][2] = -x * invz * fy;
        J[1][3] = 0;                    J[1][4] = -invz * fy;                  J[1][5] = y * invz_2 * fy;
        J[2][0] = J[0][0] - bf * y * invz_2; J[2][1] = J[0][1] + bf * x * invz_2; J[2][2] = J[0][2];
        J[2][3] = J[0][3];              J[2][4] = 0;                           J[2][5] = J[0][5] - bf * invz_2;
    } else {
        const double z = p[2];
        // -projectJac(xyz) * SE3deriv   (src/OptimizableTypes.cpp:49-63, Pinhole.cpp:71-81)
        const double pj[2][3] = {{c.fx / z, 0.0, -c.fx * x / (z * z)}, {0.0, c.fy / z, -c.fy * y / (z * z)}};
        const double D[3][6] = {{0, z, -y, 1, 0, 0}, {-z, 0, x, 0, 1, 0}, {y, -x, 0, 0, 0, 1}};
        for (int r = 0; r < 2; ++r)
            for (int k = 0; k < 6; ++k) {
                const double npj[3] = {-pj[r][0], -pj[r][1], -pj[r][2]};
                J[r][k] = npj[0] * D[0][k] + npj[1] * D[1][k] + npj[2] * D[2][k];
            }
        for (int k = 0; k < 6; ++k) J[2][k] = 0;
    }
}

// Dense LDL^T solve of the 6x6 system (Eigen::LDLT with its diagonal pivoting), isPositive() check.
// A NaN pivot (an edge on the camera plane makes H NaN) is neither positive nor negative for Eigen's sign tracking: isPositive() stays
// true and the step comes out NaN (Eigen zeroes that row of D^-1, the triangular solves with NaN in L still spread it).
bool solve6(const double Hin[6][6], const double bin[6], double x[6]) {
    double A[6][6]; int perm[6];
    for (int i = 0; i < 6; ++i) { perm[i] = i; for (int j = 0; j < 6; ++j) A[i][j] = Hin[i][j]; }
    bool positive = true, negative = true;
    for (int k = 0; k < 6; ++k) {
        int piv = k; double best = std::fabs(A[k][k]);
        for (int i = k + 1; i < 6; ++i) if (std::fabs(A[i][i]) > best) { best = std::fabs(A[i][i]); piv = i; }
        if (piv != k) {
            for (int j = 0; j < 6; ++j) std::swap(A[k][j], A[piv][j]);
            for (int i = 0; i < 6; ++i) std::swap(A[i][k], A[i][piv]);
            std::swap(perm[k], perm[piv]);
        }
        const double d = A[k][k];
        if (d > 0) negative = false; else if (d < 0) positive = false;
        if (d == 0) { positive = negative = true; break; }   // Eigen stops at an exact zero pivot (remaining block zeroed)
        for (int i = k + 1; i < 6; ++i) A[i][k] /= d;
        for (int i = k + 1; i < 6; ++i)
            for (int j = k + 1; j <= i; ++j) { A[i][j] -= A[i][k] * d * A[j][k]; A[j][i] = A[i][j]; }
    }
    if (!positive) return false;
    double y[6];
    for (int i = 0; i < 6; ++i) y[i] = bin[perm[i]];
    for (int i = 0; i < 6; ++i) for (int j = 0; j < i; ++j) y[i] -= A[i][j] * y[j];
    for (int i = 0; i < 6; ++i) y[i] = (A[i][i] != 0) ? y[i] / A[i][i] : 0.0;
    for (int i = 5; i >= 0; --i) for (int j = i + 1; j < 6; ++j) y[i] -= A[j][i] * y[j];
    for (int i = 0; i < 6; ++i) x[perm[i]] = y[i];
    return true;
}

#ifdef ORC_POSE_STUDY
struct LM;
void study_build_system(LM& lm, double H[6][6], double b[6]);
bool study_solve6(const double H[6][6], const double b[6], double x[6]);
#endif

// What one call did (orc_pose_optimize_trace): the paths it took and how close each discrete decision came to going the other way.
// Margins: |rho| for the accept / reject test (rho is already a ratio), |(ini - cur) * 1e3 - ini| / |ini| for the stop test and
// |chi2 - threshold| / threshold for the outlier classification.  Decisions that do not depend on rounding (no active edge, a failed
// solve, a non-finite value) are not counted.
struct PoseTrace {
    int rounds, iters[4];                                   // rounds run, LM iterations of each round
    int rejected, max_reject_run;                           // rejected trials in all; most consecutive rejections in one iteration
    int term_qmax, term_rho0, term_nbad, term_iters;        // how each round's optimize() ended: qmax == 10, rho == 0, n_bad >= 3, 10 iterations
    int any_sincos, empty_rounds;                           // a trial step with theta^2 >= 0.25; rounds that began with no active edge
    int max_accepted_trial;                                 // highest trial index (0-based, within an iteration) that was accepted
    double min_rho_margin, min_stop_margin, min_chi2_margin;
};

inline void margin(double& m, double dist, double scale) {
    if (std::isfinite(dist) && std::isfinite(scale) && scale != 0) m = std::min(m, std::fabs(dist) / std::fabs(scale));
}

struct LM {
    std::vector<Edge>& edges;
    const Cam& cam;
    double delta_mono, delta_stereo; float dsqr_mono, dsqr_stereo;
    SE3 est;
    double lambda = -1, ni = 2; int n_bad = 0;
    PoseTrace* tr = nullptr;

    void compute_active_errors() { for (Edge& e : edges) if (e.level == 0) edge_error(e, est, cam); }
    double active_robust_chi2() const {
        double chi = 0, rho[3];
        for (const Edge& e : edges) {
            if (e.level != 0) continue;
            if (e.robust) { huber(edge_chi2(e), e.stereo ? delta_stereo : delta_mono, e.stereo ? dsqr_stereo : dsqr_mono, rho); chi += rho[0]; }
            else chi += edge_chi2(e);
        }
        return chi;
    }
    void build_system(double H[6][6], double b[6]) {
        for (int i = 0; i < 6; ++i) { b[i] = 0; for (int j = 0; j < 6; ++j) H[i][j] = 0; }
        for (const Edge& e : edges) {
            if (e.level != 0) continue;
            double J[3][6];
            edge_jacobian(e, est, cam, J);
            const int d = e.stereo ? 3 : 2;
            double w = 1.0;
            if (e.robust) { double rho[3]; huber(edge_chi2(e), e.stereo ? delta_stereo : delta_mono, e.stereo ? dsqr_stereo : dsqr_mono, rho); w = rho[1]; }
            for (int i = 0; i < 6; ++i) {
                double s = 0;
                for (int r = 0; r < d; ++r) s += J[r][i] * (e.info * e.err[r]);
                b[i] -= w * s;
                for (int j = 0; j < 6; ++j) {
                    double h = 0;
                    for (int r = 0; r < d; ++r) h += J[r][i] * (w * e.info) * J[r][j];
                    H[i][j] += h;
                }
            }
        }
    }
    // returns true = OK, false = Terminate
    bool solve_iteration(int iteration) {
        compute_active_errors();
        double current = active_robust_chi2(), temp = current;
        const double ini = current;
        double H[6][6], b[6];
#ifdef ORC_POSE_STUDY      // tests/tools/pose_precision_study.cpp only (alternative arithmetic for the normal equations); never set for liborb_oracle.so
        study_build_system(*this, H, b);
#else
        build_system(H, b);
#endif
        if (iteration == 0) {
            double mx = 0;
            for (int j = 0; j < 6; ++j) mx = std::max(std::fabs(H[j][j]), mx);
            lambda = 1e-5 * mx; ni = 2; n_bad = 0;
        }
        double rho = 0; int qmax = 0, run = 0;
        do {
            const SE3 backup = est;
            double Hl[6][6];
            for (int i = 0; i < 6; ++i) for (int j = 0; j < 6; ++j) Hl[i][j] = H[i][j] + (i == j ? lambda : 0.0);
            double x[6] = {0, 0, 0, 0, 0, 0};
#ifdef ORC_POSE_STUDY
            const bool ok2 = study_solve6(Hl, b, x);
#else
            const bool ok2 = solve6(Hl, b, x);
#endif
            if (tr && x[0] * x[0] + x[1] * x[1] + x[2] * x[2] >= 0.25) tr->any_sincos = 1;
            est = se3_mul(se3_exp(x), est);
            compute_active_errors();
            temp = active_robust_chi2();
            if (!ok2) temp = std::numeric_limits<double>::max();
            rho = current - temp;
            double scale = 0;
            for (int j = 0; j < 6; ++j) scale += x[j] * (lambda * x[j] + b[j]);
            scale += 1e-3;
            rho /= scale;
            if (tr && ok2 && !(current == 0 && temp == 0) && std::isfinite(rho)) tr->min_rho_margin = std::min(tr->min_rho_margin, std::fabs(rho));
            if (rho > 0 && std::isfinite(temp)) {
                double alpha = 1. - std::pow((2 * rho - 1), 3);
                alpha = std::min(alpha, 2. / 3.);
                const double sf = std::max(1. / 3., alpha);
                lambda *= sf; ni = 2; current = temp;
                if (tr) { tr->max_reject_run = std::max(tr->max_reject_run, run); tr->max_accepted_trial = std::max(tr->max_accepted_trial, qmax); }
                run = 0;
            } else {
                lambda *= ni; ni *= 2; est = backup;
                if (tr) { tr->rejected += 1; tr->max_reject_run = std::max(tr->max_reject_run, ++run); }
            }
            ++qmax;
        } while (rho < 0 && qmax < 10);
        if (qmax == 10 || rho == 0) {
            if (tr) (qmax == 10 ? tr->term_qmax : tr->term_rho0) += 1;
            return false;
        }
        if (tr && ini != 0) margin(tr->min_stop_margin, (ini - current) * 1e3 - ini, ini);
        if ((ini - current) * 1e3 < ini) ++n_bad; else n_bad = 0;
        if (n_bad >= 3) {
            if (tr) tr->term_nbad += 1;
            return false;
        }
        return true;
    }
    int optimize(int iterations) {
        bool any = false;
        for (const Edge& e : edges) if (e.level == 0) { any = true; break; }
        if (tr && !any) tr->empty_rounds += 1;      // g2o keeps the vertex active even with no active edges; H = 0 -> LDLT not positive -> rho = 0 path
        bool ok = true;
        int i = 0;
        for (; i < iterations && ok; ++i) ok = solve_iteration(i);
        if (tr && ok) tr->term_iters += 1;
        return i;
    }
};

int pose_optimize(const float pose_in[7], int n, const float* xw, const float* obs, const float* inv_sigma2, const uint8_t* stereo,
                  float fx, float fy, float cx, float cy, float bf, float pose_out[7], uint8_t* outlier, PoseTrace* tr) {
    for (int i = 0; i < 7; ++i) pose_out[i] = pose_in[i];
    if (n < 3) return 0;
    std::vector<Edge> edges(n);
    for (int i = 0; i < n; ++i) {
        Edge& e = edges[i];
        for (int k = 0; k < 3; ++k) { e.xw[k] = xw[3 * i + k]; e.obs[k] = obs[3 * i + k]; }
        e.info = inv_sigma2[i]; e.stereo = stereo[i] != 0;
        outlier[i] = 0;
    }
    const Cam cam = {fx, fy, cx, cy, bf};
    const float delta_mono = std::sqrt(5.991), delta_stereo = std::sqrt(7.815);      // src/Optimizer.cc:852-853
    LM lm{edges, cam, delta_mono, delta_stereo, (float)((double)delta_mono * delta_mono), (float)((double)delta_stereo * delta_stereo)};
    lm.tr = tr;
    SE3 init;
    init.r = {pose_in[0], pose_in[1], pose_in[2], pose_in[3]};
    init.t[0] = pose_in[4]; init.t[1] = pose_in[5]; init.t[2] = pose_in[6];
    normalize_rotation(init);
    lm.est = init;
    const float chi2_mono = 5.991f, chi2_stereo = 7.815f;
    int n_bad = 0;
    for (int it = 0; it < 4; ++it) {
        lm.est = init;
        const int iters = lm.optimize(10);
        if (tr) { tr->iters[it] = iters; tr->rounds = it + 1; }
        n_bad = 0;
        for (int i = 0; i < n; ++i) {
            Edge& e = edges[i];
            if (outlier[i]) edge_error(e, lm.est, cam);
            const float chi2 = (float)edge_chi2(e);
            const float thr = e.stereo ? chi2_stereo : chi2_mono;
            if (tr) margin(tr->min_chi2_margin, (double)chi2 - thr, thr);
            if (chi2 > thr) { outlier[i] = 1; e.level = 1; ++n_bad; }
            else { outlier[i] = 0; e.level = 0; }
            if (it == 2) e.robust = false;
        }
        if (n < 10) break;
    }
    // Sophus::SE3<float> pose(rotation().cast<float>(), translation().cast<float>()) (src/Optimizer.cc:1108-1110): the SO3f quaternion
    // constructor normalises in float, coeffs /= norm (so3.hpp:481-487, 297-303; Eigen's 4-term squared norm = (x2 + y2) + (z2 + w2))
    float qf[4] = {(float)lm.est.r.x, (float)lm.est.r.y, (float)lm.est.r.z, (float)lm.est.r.w};
    const float length = std::sqrt((qf[0] * qf[0] + qf[1] * qf[1]) + (qf[2] * qf[2] + qf[3] * qf[3]));
    for (int i = 0; i < 4; ++i) pose_out[i] = qf[i] / length;
    pose_out[4] = (float)lm.est.t[0]; pose_out[5] = (float)lm.est.t[1]; pose_out[6] = (float)lm.est.t[2];
    return n - n_bad;
}

}  // namespace

extern "C" {

// pose = (qx, qy, qz, qw, tx, ty, tz) float (Sophus::SE3f of Frame::GetPose()).  Edges in keypoint order i:
// xw (3 floats, MapPoint::GetWorldPos()), obs = (kpUn.x, kpUn.y, uRight) floats, inv_sigma2 float, stereo = (uRight >= 0).
// outlier[i] written like pFrame->mvbOutlier.  Returns nInitialCorrespondences - nBad (0 if < 3 correspondences).
int orc_pose_optimize(const float pose_in[7], int n, const float* xw, const float* obs, const float* inv_sigma2,
                      const uint8_t* stereo, float fx, float fy, float cx, float cy, float bf,
                      float pose_out[7], uint8_t* outlier) {
    return pose_optimize(pose_in, n, xw, obs, inv_sigma2, stereo, fx, fy, cx, cy, bf, pose_out, outlier, nullptr);
}

// orc_pose_optimize with the same arithmetic and outputs, plus what the call did (PoseTrace above)
int orc_pose_optimize_trace(const float pose_in[7], int n, const float* xw, const float* obs, const float* inv_sigma2,
                            const uint8_t* stereo, float fx, float fy, float cx, float cy, float bf,
                            float pose_out[7], uint8_t* outlier, PoseTrace* tr) {
    *tr = PoseTrace{};
    tr->min_rho_margin = tr->min_stop_margin = tr->min_chi2_margin = std::numeric_limits<double>::infinity();
    return pose_optimize(pose_in, n, xw, obs, inv_sigma2, stereo, fx, fy, cx, cy, bf, pose_out, outlier, tr);
}

}  // extern "C"

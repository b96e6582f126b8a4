// Optimizer::LocalBundleAdjustment's numerical core (src/Optimizer.cc:1116-1499) on the device: g2o's Levenberg-Marquardt
// (Thirdparty/g2o/g2o/core/optimization_algorithm_levenberg.cpp:61-201) over key-frame poses (SE3, 6 dof) and map points
// (marginalised, 3 dof) with the Schur-complement block solver (core/block_solver.hpp:354-486), Huber kernels, the mono edge
// of src/OptimizableTypes.cpp:139-160 and the stereo edge of types/types_six_dof_expmap.cpp:190-274.  FP64.
//
// Mapping: the graph is static, so the host sorts the edges once by point and by pose (CSR); per LM iteration
//   ba_linearize   thread per edge : error, Huber weight, Jacobians -> per-edge blocks J_l^T W J_l, J_p^T W J_p, J_p^T W J_l, gradients
//   ba_point_sum   thread per point: H_ll, b_l   = ordered sums over the point's edges (deterministic)
//   ba_pose_sum    warp per pose   : H_pp, b_p   = fixed-tree sums over the pose's edges (deterministic)
// and per LM trial (lambda)
//   ba_schur       thread per point: D^-1 = (H_ll + lambda I)^-1; S -= B_i D^-1 B_j^T for the pose pairs of the point (atomicAdd into
//                                    the dense reduced system, 6 n_opt squared), coefficients += B_i D^-1 b_l
//   ba_cholesky    one CTA         : dense Cholesky of S, solve for the pose increments
//   ba_update      thread per point / pose: landmark increments by back substitution, trial estimates, gain denominator terms
//   ba_errors      thread per edge : errors and robust chi2 at the trial estimates
// The accept / reject decision needs three scalars per trial; they are read back (one small D2H + sync per trial): local BA runs
// in the mapping thread, off the per-frame latency path.
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "rgbl_ctx.h"

namespace rgbl {
namespace {

struct Se3d { double qx, qy, qz, qw, tx, ty, tz; };

__device__ __forceinline__ void q_rotate(const Se3d& q, const double v[3], double out[3]) {
    double uv[3] = {q.qy * v[2] - q.qz * v[1], q.qz * v[0] - q.qx * v[2], q.qx * v[1] - q.qy * v[0]};
    uv[0] += uv[0]; uv[1] += uv[1]; uv[2] += uv[2];
    const double c[3] = {q.qy * uv[2] - q.qz * uv[1], q.qz * uv[0] - q.qx * uv[2], q.qx * uv[1] - q.qy * uv[0]};
    out[0] = v[0] + q.qw * uv[0] + c[0]; out[1] = v[1] + q.qw * uv[1] + c[1]; out[2] = v[2] + q.qw * uv[2] + c[2];
}
__device__ __forceinline__ void se3_map(const Se3d& T, const double p[3], double out[3]) {
    q_rotate(T, p, out);
    out[0] += T.tx; out[1] += T.ty; out[2] += T.tz;
}
__device__ __forceinline__ void normalize_rotation(Se3d& T) {
    if (T.qw < 0) { T.qx *= -1; T.qy *= -1; T.qz *= -1; T.qw *= -1; }
    const double inv = rsqrt(T.qx * T.qx + T.qy * T.qy + T.qz * T.qz + T.qw * T.qw);
    T.qx *= inv; T.qy *= inv; T.qz *= inv; T.qw *= inv;
}
// SE3Quat::exp (types/se3quat.h:214-254) in closed form: q = (omega sin(th/2)/th, cos(th/2)), V = I + b Omega + c Omega^2
__device__ void se3_exp(const double* u, Se3d& T) {
    const double om[3] = {u[0], u[1], u[2]}, up[3] = {u[3], u[4], u[5]};
    const double t2 = om[0] * om[0] + om[1] * om[1] + om[2] * om[2];
    double qs, qc, b, c;
    if (t2 < 1e-10) { qs = 0.5 - t2 / 48.0; qc = 1.0 - t2 / 8.0; b = 0.5 - t2 / 24.0; c = 1.0 / 6.0 - t2 / 120.0; }
    else {
        const double th = sqrt(t2), it = 1.0 / th;
        double sh, ch;
        sincos(0.5 * th, &sh, &ch);
        qs = sh * it; qc = ch; b = 2 * sh * sh * it * it; c = (th - 2 * sh * ch) * it * it * it;
    }
    const double O[3][3] = {{0, -om[2], om[1]}, {om[2], 0, -om[0]}, {-om[1], om[0], 0}};
    double V[3][3];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            const double o2 = O[i][0] * O[0][j] + O[i][1] * O[1][j] + O[i][2] * O[2][j];
            V[i][j] = (i == j ? 1.0 : 0.0) + b * O[i][j] + c * o2;
        }
    T.qx = om[0] * qs; T.qy = om[1] * qs; T.qz = om[2] * qs; T.qw = qc;
    T.tx = V[0][0] * up[0] + V[0][1] * up[1] + V[0][2] * up[2];
    T.ty = V[1][0] * up[0] + V[1][1] * up[1] + V[1][2] * up[2];
    T.tz = V[2][0] * up[0] + V[2][1] * up[1] + V[2][2] * up[2];
    normalize_rotation(T);
}
__device__ void se3_mul(const Se3d& a, const Se3d& b, Se3d& r) {
    const double bt[3] = {b.tx, b.ty, b.tz};
    double rt[3];
    q_rotate(a, bt, rt);
    r.tx = a.tx + rt[0]; r.ty = a.ty + rt[1]; r.tz = a.tz + rt[2];
    r.qw = a.qw * b.qw - a.qx * b.qx - a.qy * b.qy - a.qz * b.qz;
    r.qx = a.qw * b.qx + a.qx * b.qw + a.qy * b.qz - a.qz * b.qy;
    r.qy = a.qw * b.qy + a.qy * b.qw + a.qz * b.qx - a.qx * b.qz;
    r.qz = a.qw * b.qz + a.qz * b.qw + a.qx * b.qy - a.qy * b.qx;
    normalize_rotation(r);
}

struct BaDev {
    int n_poses, n_opt, n_points, n_edges;
    float fx, fy, cx, cy, bf;
    const int* e_point; const int* e_pose; const float* obs; const uint8_t* stereo; const float* info;
    const int* pose_slot;                       // per pose: slot in the reduced system or -1 (fixed)
    const int* pt_start; const int* pt_edges;   // CSR: edges of a point
    const int* ps_start; const int* ps_edges;   // CSR: edges of a non-fixed pose (by slot)
};

constexpr int kEdgeBlk = 54;                    // per-edge doubles: A(6) gl(3) B(21) gp(6) Hpl(18)

// reprojection error of one edge (stereo: float 1/z as g2o's cam_project; mono: Pinhole::project)
__device__ __forceinline__ void edge_error(const BaDev& g, int k, const Se3d* poses, const double* pts, double pc[3], double e[3]) {
    const int pi = g.e_pose[k], li = g.e_point[k];
    const double X[3] = {pts[3 * li], pts[3 * li + 1], pts[3 * li + 2]};
    se3_map(poses[pi], X, pc);
    const double fx = g.fx, fy = g.fy, cx = g.cx, cy = g.cy, bf = g.bf;
    if (g.stereo[k]) {
        const float invz = (float)(1.0 / pc[2]);
        const double u = pc[0] * invz * fx + cx, v = pc[1] * invz * fy + cy;
        e[0] = (double)g.obs[3 * k] - u; e[1] = (double)g.obs[3 * k + 1] - v; e[2] = (double)g.obs[3 * k + 2] - (u - bf * invz);
    } else {
        e[0] = (double)g.obs[3 * k] - (fx * pc[0] / pc[2] + cx);
        e[1] = (double)g.obs[3 * k + 1] - (fy * pc[1] / pc[2] + cy);
        e[2] = 0;
    }
}
__device__ __forceinline__ void huber(double e2, bool stereo, double& rho0, double& rho1) {
    const double delta = stereo ? (double)(float)sqrt(7.815) : (double)(float)sqrt(5.991);
    const float dsqr = (float)(delta * delta);
    if (e2 <= (double)dsqr) { rho0 = e2; rho1 = 1.0; }
    else { const double sq = sqrt(e2); rho0 = 2 * sq * delta - (double)dsqr; rho1 = delta / sq; }
}

// block-wide deterministic sum of one double per thread into partial[blockIdx.x]
__device__ __forceinline__ void block_sum_to(double v, double* partial) {
    __shared__ double sm[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    if (lane == 0) sm[warp] = v;
    __syncthreads();
    if (warp == 0) {
        double s = lane < (int)(blockDim.x >> 5) ? sm[lane] : 0.0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
        if (lane == 0) partial[blockIdx.x] = s;
    }
}

__global__ void __launch_bounds__(128) ba_errors_kernel(BaDev g, const Se3d* __restrict__ poses, const double* __restrict__ pts,
                                                        double* __restrict__ err, double* __restrict__ partial) {
    const int k = blockIdx.x * 128 + threadIdx.x;
    double chi = 0;
    if (k < g.n_edges) {
        double pc[3], e[3];
        edge_error(g, k, poses, pts, pc, e);
        err[3 * (size_t)k] = e[0]; err[3 * (size_t)k + 1] = e[1]; err[3 * (size_t)k + 2] = e[2];
        const double info = (double)g.info[k];
        double r1;
        huber(info * (e[0] * e[0] + e[1] * e[1] + e[2] * e[2]), g.stereo[k] != 0, chi, r1);
    }
    block_sum_to(chi, partial);
}

__global__ void __launch_bounds__(128) ba_linearize_kernel(BaDev g, const Se3d* __restrict__ poses, const double* __restrict__ pts,
                                                           double* __restrict__ err, double* __restrict__ blk, double* __restrict__ partial) {
    const int k = blockIdx.x * 128 + threadIdx.x;
    double chi = 0;
    if (k < g.n_edges) {
        double pc[3], e[3];
        edge_error(g, k, poses, pts, pc, e);
        err[3 * (size_t)k] = e[0]; err[3 * (size_t)k + 1] = e[1]; err[3 * (size_t)k + 2] = e[2];
        const bool st = g.stereo[k] != 0;
        const double info = (double)g.info[k];
        double w;
        huber(info * (e[0] * e[0] + e[1] * e[1] + e[2] * e[2]), st, chi, w);
        const Se3d T = poses[g.e_pose[k]];
        double R[3][3];
        {
            const double tx = 2 * T.qx, ty = 2 * T.qy, tz = 2 * T.qz, twx = tx * T.qw, twy = ty * T.qw, twz = tz * T.qw,
                         txx = tx * T.qx, txy = ty * T.qx, txz = tz * T.qx, tyy = ty * T.qy, tyz = tz * T.qy, tzz = tz * T.qz;
            R[0][0] = 1 - (tyy + tzz); R[0][1] = txy - twz; R[0][2] = txz + twy;
            R[1][0] = txy + twz; R[1][1] = 1 - (txx + tzz); R[1][2] = tyz - twx;
            R[2][0] = txz - twy; R[2][1] = tyz + twx; R[2][2] = 1 - (txx + tyy);
        }
        const double x = pc[0], y = pc[1], z = pc[2], iz = 1.0 / z, iz2 = iz * iz;
        const double fx = g.fx, fy = g.fy, bf = st ? (double)g.bf : 0.0;
        double Jl[3][3], Jp[3][6];
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            Jl[0][c] = -fx * R[0][c] * iz + fx * x * R[2][c] * iz2;
            Jl[1][c] = -fy * R[1][c] * iz + fy * y * R[2][c] * iz2;
            Jl[2][c] = st ? Jl[0][c] - bf * R[2][c] * iz2 : 0.0;
        }
        Jp[0][0] = x * y * iz2 * fx; Jp[0][1] = -(1 + x * x * iz2) * fx; Jp[0][2] = y * iz * fx; Jp[0][3] = -iz * fx; Jp[0][4] = 0; Jp[0][5] = x * iz2 * fx;
        Jp[1][0] = (1 + y * y * iz2) * fy; Jp[1][1] = -x * y * iz2 * fy; Jp[1][2] = -x * iz * fy; Jp[1][3] = 0; Jp[1][4] = -iz * fy; Jp[1][5] = y * iz2 * fy;
        Jp[2][0] = st ? Jp[0][0] - bf * y * iz2 : 0.0; Jp[2][1] = st ? Jp[0][1] + bf * x * iz2 : 0.0; Jp[2][2] = st ? Jp[0][2] : 0.0;
        Jp[2][3] = st ? Jp[0][3] : 0.0; Jp[2][4] = 0; Jp[2][5] = st ? Jp[0][5] - bf * iz2 : 0.0;
        const double wi = w * info;
        const double we[3] = {-wi * e[0], -wi * e[1], -wi * e[2]};
        double* o = blk + (size_t)k * kEdgeBlk;
        int t = 0;
#pragma unroll
        for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = i; j < 3; ++j) o[t++] = wi * (Jl[0][i] * Jl[0][j] + Jl[1][i] * Jl[1][j] + Jl[2][i] * Jl[2][j]);
#pragma unroll
        for (int i = 0; i < 3; ++i) o[t++] = Jl[0][i] * we[0] + Jl[1][i] * we[1] + Jl[2][i] * we[2];
#pragma unroll
        for (int i = 0; i < 6; ++i)
#pragma unroll
            for (int j = i; j < 6; ++j) o[t++] = wi * (Jp[0][i] * Jp[0][j] + Jp[1][i] * Jp[1][j] + Jp[2][i] * Jp[2][j]);
#pragma unroll
        for (int i = 0; i < 6; ++i) o[t++] = Jp[0][i] * we[0] + Jp[1][i] * we[1] + Jp[2][i] * we[2];
#pragma unroll
        for (int i = 0; i < 6; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) o[t++] = wi * (Jp[0][i] * Jl[0][j] + Jp[1][i] * Jl[1][j] + Jp[2][i] * Jl[2][j]);
    }
    block_sum_to(chi, partial);
}

// H_ll (6 unique) and b_l (3) per point: ordered sum over the point's edges
__global__ void __launch_bounds__(128) ba_point_sum_kernel(BaDev g, const double* __restrict__ blk, double* __restrict__ Hll, double* __restrict__ bl) {
    const int l = blockIdx.x * 128 + threadIdx.x;
    if (l >= g.n_points) return;
    double a[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = g.pt_start[l]; i < g.pt_start[l + 1]; ++i) {
        const double* o = blk + (size_t)g.pt_edges[i] * kEdgeBlk;
#pragma unroll
        for (int t = 0; t < 9; ++t) a[t] += o[t];
    }
#pragma unroll
    for (int t = 0; t < 6; ++t) Hll[6 * (size_t)l + t] = a[t];
#pragma unroll
    for (int t = 0; t < 3; ++t) bl[3 * (size_t)l + t] = a[6 + t];
}

// H_pp (21 unique) and b_p (6) per non-fixed pose: one CTA per pose, threads stride the pose's edges (a key frame sees
// thousands of points), fixed reduction tree (shuffles inside a warp, then the 8 warp sums in order): deterministic
__global__ void __launch_bounds__(256) ba_pose_sum_kernel(BaDev g, const double* __restrict__ blk, double* __restrict__ Hpp, double* __restrict__ bp) {
    __shared__ double sm[8][27];
    const int s = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double a[27];
#pragma unroll
    for (int t = 0; t < 27; ++t) a[t] = 0;
    for (int i = g.ps_start[s] + threadIdx.x; i < g.ps_start[s + 1]; i += 256) {
        const double* o = blk + (size_t)g.ps_edges[i] * kEdgeBlk + 9;
#pragma unroll
        for (int t = 0; t < 27; ++t) a[t] += o[t];
    }
#pragma unroll
    for (int t = 0; t < 27; ++t) {
        double v = a[t];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
        if (lane == 0) sm[warp][t] = v;
    }
    __syncthreads();
    if (threadIdx.x < 27) {
        double v = 0;
#pragma unroll
        for (int w = 0; w < 8; ++w) v += sm[w][threadIdx.x];
        if (threadIdx.x < 21) Hpp[21 * (size_t)s + threadIdx.x] = v; else bp[6 * (size_t)s + (threadIdx.x - 21)] = v;
    }
}

// max |diagonal| over all free vertices (lambda init)
__global__ void __launch_bounds__(256) ba_maxdiag_kernel(BaDev g, const double* __restrict__ Hpp, const double* __restrict__ Hll, double* __restrict__ out) {
    __shared__ double sm[256];
    double m = 0;
    for (int i = threadIdx.x; i < g.n_opt * 6; i += 256) { const int s = i / 6, j = i % 6; m = fmax(m, fabs(Hpp[21 * (size_t)s + (j * 6 - (j * (j - 1)) / 2)])); }
    for (int i = threadIdx.x; i < g.n_points * 3; i += 256) { const int l = i / 3, j = i % 3; m = fmax(m, fabs(Hll[6 * (size_t)l + (j == 0 ? 0 : (j == 1 ? 3 : 5))])); }
    sm[threadIdx.x] = m;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) sm[threadIdx.x] = fmax(sm[threadIdx.x], sm[threadIdx.x + o]); __syncthreads(); }
    if (threadIdx.x == 0) *out = sm[0];
}

__device__ __forceinline__ bool dinv3(const double* h6, double lam, double D[9]) {
    const double a = h6[0] + lam, b = h6[1], c = h6[2], e = h6[3] + lam, f = h6[4], i = h6[5] + lam;     // symmetric: [a b c; b e f; c f i]
    const double det = a * (e * i - f * f) - b * (b * i - f * c) + c * (b * f - e * c);
    const double id = 1.0 / det;
    D[0] = (e * i - f * f) * id; D[1] = (c * f - b * i) * id; D[2] = (b * f - c * e) * id;
    D[3] = D[1]; D[4] = (a * i - c * c) * id; D[5] = (c * b - a * f) * id;
    D[6] = D[2]; D[7] = D[5]; D[8] = (a * e - b * b) * id;
    return true;
}

// S = blockdiag(H_pp) + lambda I, coefficients = 0
__global__ void __launch_bounds__(256) ba_schur_init_kernel(BaDev g, const double* __restrict__ Hpp, double lam, double* __restrict__ S, double* __restrict__ coef) {
    const int n = 6 * g.n_opt;
    const size_t tot = (size_t)n * n;
    for (size_t i = blockIdx.x * (size_t)256 + threadIdx.x; i < tot; i += (size_t)gridDim.x * 256) {
        const int r = (int)(i / n), c = (int)(i % n);
        double v = 0;
        if (r / 6 == c / 6) {
            const int s = r / 6, a = min(r % 6, c % 6), b = max(r % 6, c % 6);
            v = Hpp[21 * (size_t)s + (a * 6 - (a * (a - 1)) / 2 + (b - a))];
            if (r == c) v += lam;
        }
        S[i] = v;
        if (i < (size_t)n) coef[i] = 0;
    }
}

// one warp per point: the lanes share the m^2 pose pairs of the point (m observations)
__global__ void __launch_bounds__(128) ba_schur_kernel(BaDev g, const double* __restrict__ blk, const double* __restrict__ Hll, const double* __restrict__ bl,
                                                       double lam, double* __restrict__ S, double* __restrict__ coef) {
    const int l = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (l >= g.n_points) return;
    double D[9];
    dinv3(Hll + 6 * (size_t)l, lam, D);
    const double b0 = bl[3 * (size_t)l], b1 = bl[3 * (size_t)l + 1], b2 = bl[3 * (size_t)l + 2];
    const double db[3] = {D[0] * b0 + D[1] * b1 + D[2] * b2, D[3] * b0 + D[4] * b1 + D[5] * b2, D[6] * b0 + D[7] * b1 + D[8] * b2};
    const int n = 6 * g.n_opt, eb = g.pt_start[l], m = g.pt_start[l + 1] - eb;
    for (int i1 = lane; i1 < m; i1 += 32) {
        const int k1 = g.pt_edges[eb + i1], s1 = g.pose_slot[g.e_pose[k1]];
        if (s1 < 0) continue;
        const double* B1 = blk + (size_t)k1 * kEdgeBlk + 36;
#pragma unroll
        for (int i = 0; i < 6; ++i) atomicAdd(&coef[6 * s1 + i], B1[3 * i] * db[0] + B1[3 * i + 1] * db[1] + B1[3 * i + 2] * db[2]);
    }
    for (int t = lane; t < m * m; t += 32) {
        const int i1 = t / m, i2 = t - i1 * m;
        const int k1 = g.pt_edges[eb + i1], k2 = g.pt_edges[eb + i2];
        const int s1 = g.pose_slot[g.e_pose[k1]], s2 = g.pose_slot[g.e_pose[k2]];
        if (s1 < 0 || s2 < 0 || s2 > s1) continue;                 // lower triangle only (the Cholesky reads it)
        const double* B1 = blk + (size_t)k1 * kEdgeBlk + 36;
        const double* B2 = blk + (size_t)k2 * kEdgeBlk + 36;
        double b2v[18];
#pragma unroll
        for (int i = 0; i < 18; ++i) b2v[i] = B2[i];
#pragma unroll
        for (int i = 0; i < 6; ++i) {
            const double a0 = B1[3 * i], a1 = B1[3 * i + 1], a2 = B1[3 * i + 2];
            const double bd0 = a0 * D[0] + a1 * D[3] + a2 * D[6], bd1 = a0 * D[1] + a1 * D[4] + a2 * D[7], bd2 = a0 * D[2] + a1 * D[5] + a2 * D[8];
#pragma unroll
            for (int j = 0; j < 6; ++j)
                atomicAdd(&S[(size_t)(6 * s1 + i) * n + 6 * s2 + j], -(bd0 * b2v[3 * j] + bd1 * b2v[3 * j + 1] + bd2 * b2v[3 * j + 2]));
        }
    }
}

// dense Cholesky S = L L^T on the lower triangle, then L L^T x = b_p - coef, by one CTA.  The matrix is staged in shared
// memory when it fits (n <= 160: 6 n_opt squared doubles), else it is factored in place in global memory.  status[0] = 1 on a
// non-positive pivot (g2o: the linear solver fails -> the LM trial is rejected).
__global__ void __launch_bounds__(1024) ba_cholesky_kernel(int n, int use_smem, double* __restrict__ Sg, const double* __restrict__ bp, const double* __restrict__ coef,
                                                           double* __restrict__ x, int* __restrict__ status) {
    extern __shared__ double s_mat[];
    const int tid = threadIdx.x, nt = blockDim.x;
    double* S = use_smem ? s_mat : Sg;
    double* y = use_smem ? s_mat + (size_t)n * n : x;
    if (use_smem) for (int i = tid; i < n * n; i += nt) S[i] = Sg[i];
    for (int i = tid; i < n; i += nt) y[i] = bp[i] - coef[i];
    __syncthreads();
    // two barriers per column: every thread reads the pivot itself (uniform failure test, no broadcast step)
    bool fail = false;
    for (int k = 0; k < n; ++k) {
        const double d = S[(size_t)k * n + k];
        if (!(d > 0) || !(d <= DBL_MAX)) { fail = true; break; }
        const double sd = sqrt(d), inv = 1.0 / sd;
        __syncthreads();                                          // everyone has read the pivot before it is overwritten
        for (int i = k + tid; i < n; i += nt) S[(size_t)i * n + k] = (i == k) ? sd : S[(size_t)i * n + k] * inv;
        __syncthreads();
        // trailing update of the lower triangle (rows i > k, columns k < j <= i) on a 16-wide thread grid: no index divisions
        const int tx = tid & 15, ty = tid >> 4, ny = nt >> 4;
        for (int i = k + 1 + ty; i < n; i += ny) {
            const double lik = S[(size_t)i * n + k];
            for (int j = k + 1 + tx; j <= i; j += 16) S[(size_t)i * n + j] -= lik * S[(size_t)j * n + k];
        }
        __syncthreads();
    }
    if (fail) { if (tid == 0) status[0] = 1; for (int i = tid; i < n; i += nt) x[i] = 0; return; }
    if (tid == 0) status[0] = 0;
    // column-oriented substitutions, one barrier per column: every thread forms y[k] / L[k][k] itself
    for (int k = 0; k < n; ++k) {
        const double yk = y[k] / S[(size_t)k * n + k];
        __syncthreads();
        if (tid == 0) y[k] = yk;
        for (int i = k + 1 + tid; i < n; i += nt) y[i] -= S[(size_t)i * n + k] * yk;
        __syncthreads();
    }
    for (int k = n - 1; k >= 0; --k) {
        const double yk = y[k] / S[(size_t)k * n + k];
        __syncthreads();
        if (tid == 0) y[k] = yk;
        for (int i = tid; i < k; i += nt) y[i] -= S[(size_t)k * n + i] * yk;
        __syncthreads();
    }
    if (use_smem) for (int i = tid; i < n; i += nt) x[i] = y[i];
}

// landmark increments, trial points, gain denominator terms of the landmarks.  After a failed factorisation (status[0] != 0) the whole
// solution is zero: g2o's solve() (core/block_solver.hpp:354-486) returns when the reduced system cannot be solved, before the landmark
// back substitution.  The trial points are then the current ones, so the errors the rejected trial leaves behind (the erase test reads
// them) are those of the estimate, and no increment is formed from a D^-1 that need not be finite
__global__ void __launch_bounds__(128) ba_point_update_kernel(BaDev g, const double* __restrict__ blk, const double* __restrict__ Hll, const double* __restrict__ bl,
                                                              double lam, const double* __restrict__ xp, const int* __restrict__ status,
                                                              const double* __restrict__ pts, double* __restrict__ pts_try, double* __restrict__ partial) {
    const int l = blockIdx.x * 128 + threadIdx.x;
    double sc = 0;
    if (l < g.n_points && status[0] != 0) {
#pragma unroll
        for (int i = 0; i < 3; ++i) pts_try[3 * (size_t)l + i] = pts[3 * (size_t)l + i];
    } else if (l < g.n_points) {
        double D[9];
        dinv3(Hll + 6 * (size_t)l, lam, D);
        double c[3] = {bl[3 * (size_t)l], bl[3 * (size_t)l + 1], bl[3 * (size_t)l + 2]};
        for (int i1 = g.pt_start[l]; i1 < g.pt_start[l + 1]; ++i1) {
            const int k = g.pt_edges[i1], s = g.pose_slot[g.e_pose[k]];
            if (s < 0) continue;
            const double* B = blk + (size_t)k * kEdgeBlk + 36;
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                double v = 0;
#pragma unroll
                for (int i = 0; i < 6; ++i) v += B[3 * i + j] * xp[6 * s + i];
                c[j] -= v;
            }
        }
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const double xl = D[3 * i] * c[0] + D[3 * i + 1] * c[1] + D[3 * i + 2] * c[2];
            pts_try[3 * (size_t)l + i] = pts[3 * (size_t)l + i] + xl;
            sc += xl * (lam * xl + bl[3 * (size_t)l + i]);
        }
    }
    block_sum_to(sc, partial);
}

__global__ void __launch_bounds__(128) ba_pose_update_kernel(BaDev g, double lam, const double* __restrict__ xp, const double* __restrict__ bp,
                                                             const Se3d* __restrict__ poses, Se3d* __restrict__ poses_try, double* __restrict__ partial) {
    const int p = blockIdx.x * 128 + threadIdx.x;
    double sc = 0;
    if (p < g.n_poses) {
        const int s = g.pose_slot[p];
        Se3d T = poses[p];
        if (s >= 0) {
            Se3d E, Tn;
            se3_exp(xp + 6 * s, E);
            se3_mul(E, T, Tn);
            T = Tn;
#pragma unroll
            for (int i = 0; i < 6; ++i) sc += xp[6 * s + i] * (lam * xp[6 * s + i] + bp[6 * s + i]);
        }
        poses_try[p] = T;
    }
    block_sum_to(sc, partial);
}

// sums n partials (fixed order) into out[slot]
__global__ void __launch_bounds__(256) ba_final_sum_kernel(const double* __restrict__ partial, int n, double* __restrict__ out) {
    __shared__ double sm[256];
    double s = 0;
    for (int i = threadIdx.x; i < n; i += 256) s += partial[i];
    sm[threadIdx.x] = s;
    __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) sm[threadIdx.x] += sm[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) *out = sm[0];
}

__global__ void __launch_bounds__(128) ba_flags_kernel(BaDev g, const Se3d* __restrict__ poses, const double* __restrict__ pts, const double* __restrict__ err,
                                                       uint8_t* __restrict__ erase) {
    const int k = blockIdx.x * 128 + threadIdx.x;
    if (k >= g.n_edges) return;
    const double info = (double)g.info[k];
    const double chi = info * (err[3 * (size_t)k] * err[3 * (size_t)k] + err[3 * (size_t)k + 1] * err[3 * (size_t)k + 1] + err[3 * (size_t)k + 2] * err[3 * (size_t)k + 2]);
    const int li = g.e_point[k];
    const double X[3] = {pts[3 * li], pts[3 * li + 1], pts[3 * li + 2]};
    double pc[3];
    se3_map(poses[g.e_pose[k]], X, pc);
    erase[k] = (chi > (g.stereo[k] ? 7.815 : 5.991) || !(pc[2] > 0.0)) ? 1 : 0;
}

__global__ void ba_init_state_kernel(int n_poses, const float* __restrict__ poses_f, Se3d* __restrict__ poses, int n3, const float* __restrict__ pts_f, double* __restrict__ pts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_poses) {
        Se3d T{poses_f[7 * i], poses_f[7 * i + 1], poses_f[7 * i + 2], poses_f[7 * i + 3], poses_f[7 * i + 4], poses_f[7 * i + 5], poses_f[7 * i + 6]};
        if (T.qw < 0) { T.qx *= -1; T.qy *= -1; T.qz *= -1; T.qw *= -1; }
        const double nrm = sqrt(T.qx * T.qx + T.qy * T.qy + T.qz * T.qz + T.qw * T.qw);
        T.qx /= nrm; T.qy /= nrm; T.qz /= nrm; T.qw /= nrm;
        poses[i] = T;
    }
    if (i < n3) pts[i] = (double)pts_f[i];
}

__global__ void ba_export_kernel(int n_poses, const Se3d* __restrict__ poses, const int* __restrict__ slot, const float* __restrict__ poses_in, float* __restrict__ poses_f,
                                 int n3, const double* __restrict__ pts, float* __restrict__ pts_f) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n_poses) {
        if (slot[i] < 0) { for (int j = 0; j < 7; ++j) poses_f[7 * i + j] = poses_in[7 * i + j]; }
        else {
            const Se3d T = poses[i];
            poses_f[7 * i] = (float)T.qx; poses_f[7 * i + 1] = (float)T.qy; poses_f[7 * i + 2] = (float)T.qz; poses_f[7 * i + 3] = (float)T.qw;
            poses_f[7 * i + 4] = (float)T.tx; poses_f[7 * i + 5] = (float)T.ty; poses_f[7 * i + 6] = (float)T.tz;
        }
    }
    if (i < n3) pts_f[i] = (float)pts[i];
}

}  // namespace
}  // namespace rgbl

using namespace rgbl;

extern "C" int rgbl_local_bundle_adjustment(rgbl_ctx* ctx, int n_poses, const float* poses, const uint8_t* pose_fixed, int n_points, const float* points,
                                            int n_edges, const int32_t* e_point, const int32_t* e_pose, const float* obs, const uint8_t* stereo,
                                            const float* inv_sigma2, float fx, float fy, float cx, float cy, float bf, int iterations,
                                            float* poses_out, float* points_out, uint8_t* edge_erase, int* iterations_run) {
    Ctx* c = reinterpret_cast<Ctx*>(ctx);
    if (const int rc = require_idle(c)) return rc;
    if (n_poses < 0 || n_points < 0 || n_edges < 0 || iterations < 0 || (n_poses && (!poses || !pose_fixed || !poses_out)) || (n_points && (!points || !points_out)) ||
        (n_edges && (!e_point || !e_pose || !obs || !stereo || !inv_sigma2 || !edge_erase))) { c->err = "bad local BA arguments"; return RGBL_E_INVALID; }
    for (int k = 0; k < n_edges; ++k)
        if (e_point[k] < 0 || e_point[k] >= n_points || e_pose[k] < 0 || e_pose[k] >= n_poses) { c->err = "local BA edge index out of range"; return RGBL_E_INVALID; }
    if (iterations_run) *iterations_run = 0;
    if (n_poses) std::memcpy(poses_out, poses, (size_t)n_poses * 7 * sizeof(float));
    if (n_points) std::memcpy(points_out, points, (size_t)n_points * 3 * sizeof(float));
    if (n_edges) std::memset(edge_erase, 0, n_edges);
    if (n_edges == 0 || n_points == 0) return RGBL_OK;
    CU(cudaSetDevice(c->cfg.device));
    cudaStream_t st = c->st;

    // ---- static structure on the host: reduced-system slots, edges by point, edges by free pose ----
    std::vector<int> slot(n_poses), pt_start(n_points + 1, 0), pt_edges(n_edges);
    int n_opt = 0;
    for (int p = 0; p < n_poses; ++p) slot[p] = pose_fixed[p] ? -1 : n_opt++;
    for (int k = 0; k < n_edges; ++k) ++pt_start[e_point[k] + 1];
    for (int l = 0; l < n_points; ++l) pt_start[l + 1] += pt_start[l];
    { std::vector<int> fill(pt_start.begin(), pt_start.end() - 1); for (int k = 0; k < n_edges; ++k) pt_edges[fill[e_point[k]]++] = k; }
    std::vector<int> ps_start(n_opt + 1, 0), ps_edges;
    for (int k = 0; k < n_edges; ++k) if (slot[e_pose[k]] >= 0) ++ps_start[slot[e_pose[k]] + 1];
    for (int s = 0; s < n_opt; ++s) ps_start[s + 1] += ps_start[s];
    ps_edges.resize(std::max(ps_start[n_opt], 1));
    { std::vector<int> fill(ps_start.begin(), ps_start.end() - 1); for (int k = 0; k < n_edges; ++k) { const int s = slot[e_pose[k]]; if (s >= 0) ps_edges[fill[s]++] = k; } }
    const int n = 6 * n_opt;
    const int eb = (n_edges + 127) / 128, pb = (n_points + 127) / 128, qb = (n_poses + 127) / 128;
    const int n_part = std::max(eb, std::max(pb, qb));

    // ---- device arena ----
    ArenaCarve a(c, (size_t)n_edges * (kEdgeBlk * 8 + 3 * 8 + 4 + 4 + 12 + 1 + 4 + 8) + (size_t)n_points * (4 + 9 * 8 * 2 + 6 * 8 + 12 + 12) + (size_t)n_poses * (2 * 56 + 8 + 2 * 28) +
                    (size_t)n_opt * (27 * 8 + 8 + 6 * 8 * 3) + (size_t)n * n * 8 + (size_t)n_part * 8 * 3 + (1 << 16));
    if (!a.base) { c->err = "device allocation failed (local BA)"; return RGBL_E_CUDA; }
    int* d_epoint = a.take<int>(n_edges); int* d_epose = a.take<int>(n_edges); float* d_obs = a.take<float>((size_t)3 * n_edges);
    uint8_t* d_stereo = a.take<uint8_t>(n_edges); float* d_info = a.take<float>(n_edges); uint8_t* d_erase = a.take<uint8_t>(n_edges);
    int* d_slot = a.take<int>(n_poses); int* d_ptstart = a.take<int>(n_points + 1); int* d_ptedges = a.take<int>(n_edges);
    int* d_psstart = a.take<int>(n_opt + 1); int* d_psedges = a.take<int>(ps_edges.size());
    float* d_poses_f = a.take<float>((size_t)7 * n_poses); float* d_pts_f = a.take<float>((size_t)3 * n_points);
    float* d_poses_o = a.take<float>((size_t)7 * n_poses); float* d_pts_o = a.take<float>((size_t)3 * n_points);
    Se3d* d_pose[2] = {a.take<Se3d>(n_poses), a.take<Se3d>(n_poses)};
    double* d_pts[2] = {a.take<double>((size_t)3 * n_points), a.take<double>((size_t)3 * n_points)};
    double* d_err = a.take<double>((size_t)3 * n_edges); double* d_blk = a.take<double>((size_t)kEdgeBlk * n_edges);
    double* d_Hll = a.take<double>((size_t)6 * n_points); double* d_bl = a.take<double>((size_t)3 * n_points);
    double* d_Hpp = a.take<double>((size_t)21 * std::max(n_opt, 1)); double* d_bp = a.take<double>((size_t)6 * std::max(n_opt, 1));
    double* d_S = a.take<double>((size_t)std::max(n, 1) * std::max(n, 1)); double* d_coef = a.take<double>(std::max(n, 1)); double* d_xp = a.take<double>(std::max(n, 1));
    double* d_part = a.take<double>((size_t)3 * n_part); double* d_scal = a.take<double>(8); int* d_status = a.take<int>(4);
    if (a.used > a.cap) { c->err = "local BA arena too small (internal)"; return RGBL_E_CUDA; }

    auto up = [&](void* d, const void* h, size_t bytes) { return cudaMemcpyAsync(d, h, bytes, cudaMemcpyHostToDevice, st); };
    CU(up(d_epoint, e_point, (size_t)n_edges * 4)); CU(up(d_epose, e_pose, (size_t)n_edges * 4)); CU(up(d_obs, obs, (size_t)n_edges * 12));
    CU(up(d_stereo, stereo, n_edges)); CU(up(d_info, inv_sigma2, (size_t)n_edges * 4)); CU(up(d_slot, slot.data(), (size_t)n_poses * 4));
    CU(up(d_ptstart, pt_start.data(), (size_t)(n_points + 1) * 4)); CU(up(d_ptedges, pt_edges.data(), (size_t)n_edges * 4));
    CU(up(d_psstart, ps_start.data(), (size_t)(n_opt + 1) * 4)); CU(up(d_psedges, ps_edges.data(), ps_edges.size() * 4));
    CU(up(d_poses_f, poses, (size_t)n_poses * 28)); CU(up(d_pts_f, points, (size_t)n_points * 12));
    CU(cudaMemsetAsync(d_status, 0, 16, st));
    CU(cudaMemsetAsync(d_err, 0, (size_t)3 * n_edges * sizeof(double), st));      // iterations = 0: the erase test sees zero errors, only depth can flag
    BaDev g{n_poses, n_opt, n_points, n_edges, fx, fy, cx, cy, bf, d_epoint, d_epose, d_obs, d_stereo, d_info, d_slot, d_ptstart, d_ptedges, d_psstart, d_psedges};
    const int init_n = std::max(n_poses, 3 * n_points);
    ba_init_state_kernel<<<(init_n + 255) / 256, 256, 0, st>>>(n_poses, d_poses_f, d_pose[0], 3 * n_points, d_pts_f, d_pts[0]);

    const size_t chol_need = ((size_t)n * n + n) * sizeof(double);
    const int chol_in_smem = chol_need <= 200 * 1024 ? 1 : 0;
    const size_t chol_smem = chol_in_smem ? chol_need : 0;
    const int chol_threads = n <= 192 ? 256 : 1024;          // small systems: cheaper barriers matter more than lanes
    {
        static bool done[64] = {};
        const int dev = c->cfg.device;
        if (dev >= 0 && dev < 64 && !done[dev]) { cudaFuncSetAttribute(ba_cholesky_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); done[dev] = true; }
    }
    double* h = reinterpret_cast<double*>(c->h_scalars.get());      // 16 pinned ints = 8 doubles
    int cur = 0, it_run = 0;
    double lambda = 0, ni = 2;
    int n_bad = 0;
    long launches = 1;
    stage_begin(c, ST_POSE, st);
    for (int it = 0; it < iterations; ++it) {
        // computeActiveErrors + activeRobustChi2 + buildSystem at the current estimates
        ba_linearize_kernel<<<eb, 128, 0, st>>>(g, d_pose[cur], d_pts[cur], d_err, d_blk, d_part);
        ba_final_sum_kernel<<<1, 256, 0, st>>>(d_part, eb, d_scal + 0);
        ba_point_sum_kernel<<<pb, 128, 0, st>>>(g, d_blk, d_Hll, d_bl);
        if (n_opt) ba_pose_sum_kernel<<<n_opt, 256, 0, st>>>(g, d_blk, d_Hpp, d_bp);
        launches += 4;
        if (it == 0) { ba_maxdiag_kernel<<<1, 256, 0, st>>>(g, d_Hpp, d_Hll, d_scal + 1); ++launches; }
        CU(cudaMemcpyAsync(h, d_scal, 2 * sizeof(double), cudaMemcpyDeviceToHost, st));
        CU(cudaStreamSynchronize(st));
        double current = h[0];
        const double ini = current;
        if (it == 0) { lambda = 1e-5 * h[1]; ni = 2; n_bad = 0; }
        double rho = 0; int qmax = 0;
        do {
            const int nxt = cur ^ 1;
            if (n_opt) {
                ba_schur_init_kernel<<<std::min((n * n + 255) / 256, 1024), 256, 0, st>>>(g, d_Hpp, lambda, d_S, d_coef);
                ba_schur_kernel<<<(n_points + 3) / 4, 128, 0, st>>>(g, d_blk, d_Hll, d_bl, lambda, d_S, d_coef);
                ba_cholesky_kernel<<<1, chol_threads, chol_smem, st>>>(n, chol_in_smem, d_S, d_bp, d_coef, d_xp, d_status);
                launches += 3;
            }
            ba_point_update_kernel<<<pb, 128, 0, st>>>(g, d_blk, d_Hll, d_bl, lambda, d_xp, d_status, d_pts[cur], d_pts[nxt], d_part);
            ba_final_sum_kernel<<<1, 256, 0, st>>>(d_part, pb, d_scal + 2);
            ba_pose_update_kernel<<<qb, 128, 0, st>>>(g, lambda, d_xp, d_bp, d_pose[cur], d_pose[nxt], d_part + n_part);
            ba_final_sum_kernel<<<1, 256, 0, st>>>(d_part + n_part, qb, d_scal + 3);
            ba_errors_kernel<<<eb, 128, 0, st>>>(g, d_pose[nxt], d_pts[nxt], d_err, d_part + 2 * n_part);
            ba_final_sum_kernel<<<1, 256, 0, st>>>(d_part + 2 * n_part, eb, d_scal + 4);
            launches += 6;
            CU(cudaMemcpyAsync(h, d_scal, 5 * sizeof(double), cudaMemcpyDeviceToHost, st));
            CU(cudaMemcpyAsync(c->h_scalars + 12, d_status, sizeof(int), cudaMemcpyDeviceToHost, st));
            CU(cudaStreamSynchronize(st));
            const bool ok2 = c->h_scalars[12] == 0;
            double temp = h[4];
            if (!ok2) temp = DBL_MAX;
            rho = current - temp;
            const double scale = h[2] + h[3] + 1e-3;
            rho /= scale;
            if (rho > 0 && std::isfinite(temp)) {
                double alpha = 1. - std::pow(2 * rho - 1, 3);
                alpha = std::min(alpha, 2. / 3.);
                lambda *= std::max(1. / 3., alpha); ni = 2; current = temp; cur = nxt;
            } else {
                lambda *= ni; ni *= 2;
            }
            ++qmax;
        } while (rho < 0 && qmax < 10);
        ++it_run;
        if (qmax == 10 || rho == 0) break;
        if ((ini - current) * 1e3 < ini) ++n_bad; else n_bad = 0;
        if (n_bad >= 3) break;
    }
    ba_flags_kernel<<<eb, 128, 0, st>>>(g, d_pose[cur], d_pts[cur], d_err, d_erase);
    ba_export_kernel<<<(init_n + 255) / 256, 256, 0, st>>>(n_poses, d_pose[cur], d_slot, d_poses_f, d_poses_o, 3 * n_points, d_pts[cur], d_pts_o);
    launches += 2;
    stage_end(c, ST_POSE, st, (int)launches);
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(poses_out, d_poses_o, (size_t)n_poses * 28, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(points_out, d_pts_o, (size_t)n_points * 12, cudaMemcpyDeviceToHost, st));
    CU(cudaMemcpyAsync(edge_erase, d_erase, n_edges, cudaMemcpyDeviceToHost, st));
    CU(cudaStreamSynchronize(st));
    prof_collect(c);
    if (iterations_run) *iterations_run = it_run;
    return RGBL_OK;
}
